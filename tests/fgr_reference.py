"""Numpy float64 restatement of Fast Global Registration as include/teaser_b200.h defines it (tzr_fgr_batch, DESIGN.md
§3.20): the normalisation, the optimiser and the transform back to the input frame, term by term.

Every sum runs in the device's order (block_sum: thread l of 256 takes items l, l + 256, ..., then a butterfly inside
each warp of 32 and the 8 warp sums in warp order), every product and sum in the header's parentheses, so the
restatement and the device differ only where sin / cos differ (the host libm against CUDA's sincos, at most an ulp or
two per call).  The 6 x 6 solve and the Euler rotation are tests/icp_plane_reference.py's.  The evaluation (fitness,
RMSE) is tzr_icp_batch's and is not restated here.
"""
from __future__ import annotations

import numpy as np

from icp_plane_reference import euler, solve6

THREADS = 256
MIN_CORR = 10


def block_sum(terms):
    """The device's fixed-order sum of the rows of terms (n, m) over a CTA of 256 threads: thread l adds rows l,
    l + 256, ... in ascending order starting from 0, a butterfly (xor 16, 8, 4, 2, 1) inside each warp, then the 8 warp
    sums in warp order from 0."""
    terms = np.asarray(terms, dtype=np.float64)
    n, m = terms.shape
    acc = np.zeros((THREADS, m))
    for k0 in range(0, n, THREADS):
        blk = terms[k0:k0 + THREADS]
        acc[:blk.shape[0]] = acc[:blk.shape[0]] + blk
    return _reduce(acc)


def _reduce(acc):
    lane = np.arange(THREADS)
    for o in (16, 8, 4, 2, 1):
        acc = acc + acc[lane ^ o]
    s = np.zeros(acc.shape[1])
    for w in range(THREADS // 32):
        s = s + acc[32 * w]
    return s


def finite_rows(a):
    return np.isfinite(a).all(axis=1)


def normalise(x, y, corr, use_absolute_scale=0):
    """(p, q, info) of the header's normalisation: the means of the finite points, sigma, scale_global and mu_start,
    and the usable correspondences (both ends finite) in input order, as float64 rows of the normalised frame."""
    x = np.asarray(x, dtype=np.float32).astype(np.float64)
    y = np.asarray(y, dtype=np.float32).astype(np.float64)
    corr = np.asarray(corr, dtype=np.int64).reshape(-1, 2)
    means, sigma = [], 0.0
    for c in (x, y):
        f = finite_rows(c)
        s = block_sum(np.where(f[:, None], np.concatenate([c, np.ones((len(c), 1))], axis=1), 0.0))
        m = s[:3] / s[3]
        means.append(m)
        d = c[f] - m
        if len(d):
            sigma = max(sigma, float(np.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]).max()))
    sg = 1.0 if use_absolute_scale or sigma == 0.0 else sigma
    mu0 = sigma if use_absolute_scale else 1.0
    X, Y = x[corr[:, 0]], y[corr[:, 1]]
    ok = finite_rows(X) & finite_rows(Y)
    p = (X[ok] - means[0]) / sg
    q = (Y[ok] - means[1]) / sg
    return p, q, dict(mean_s=means[0], mean_t=means[1], sigma=sigma, scale_global=sg, mu0=mu0, K=int(ok.sum()))


def mu_schedule(mu0, iteration_number, max_dist, division_factor=1.4, decrease_mu=1):
    """mu at every iteration: divided by division_factor when decrease_mu, itr % 4 == 0 and mu > max_dist."""
    out, mu = [], mu0
    for itr in range(iteration_number):
        if decrease_mu and itr % 4 == 0 and mu > max_dist:
            mu = mu / division_factor
        out.append(mu)
    return out


def row_terms(J, r, w):
    """icp_row_terms<true> over many rows: (w J_a) J_b for the 21 entries of the upper triangle row by row, then
    (w J_a) r; J (n, 6), r and w (n,)."""
    wJ = w[:, None] * J
    cols = [wJ[:, a] * J[:, b] for a in range(6) for b in range(a, 6)]
    cols += [wJ[:, a] * r for a in range(6)]
    return np.stack(cols, axis=1)


def system(p, q, R, t, mu):
    """The 27 sums of one iteration at T = (R, t) in the device's order: per thread, each row's x, y, z terms in that
    order."""
    K = len(p)
    qq = np.empty_like(q)
    for d in range(3):
        qq[:, d] = ((R[d, 0] * q[:, 0] + R[d, 1] * q[:, 1]) + R[d, 2] * q[:, 2]) + t[d]
    r = p - qq
    w = mu / (((r[:, 0] * r[:, 0] + r[:, 1] * r[:, 1]) + r[:, 2] * r[:, 2]) + mu)
    w = w * w
    z, one = np.zeros(K), np.ones(K)
    Jx = np.stack([z, -qq[:, 2], qq[:, 1], -one, z, z], axis=1)
    Jy = np.stack([qq[:, 2], z, -qq[:, 0], z, -one, z], axis=1)
    Jz = np.stack([-qq[:, 1], qq[:, 0], z, z, z, -one], axis=1)
    tx, ty, tz = row_terms(Jx, r[:, 0], w), row_terms(Jy, r[:, 1], w), row_terms(Jz, r[:, 2], w)
    acc = np.zeros((THREADS, 27))
    for k0 in range(0, K, THREADS):
        n = min(THREADS, K - k0)
        acc[:n] = ((acc[:n] + tx[k0:k0 + n]) + ty[k0:k0 + n]) + tz[k0:k0 + n]
    return _reduce(acc), w


def unpack(v):
    """(A, g) from the 27 sums."""
    A = np.zeros((6, 6))
    k = 0
    for a in range(6):
        for b in range(a, 6):
            A[a, b] = A[b, a] = v[k]
            k += 1
    return A, v[21:]


def step(R, t, xi):
    """T <- Delta T T with Delta R = Rz(xi2) Ry(xi1) Rx(xi0), each entry ((a b + c d) + e f) (+ xi)."""
    D = euler(*xi[:3])
    Rn, tn = np.empty((3, 3)), np.empty(3)
    for r in range(3):
        for c in range(3):
            Rn[r, c] = (D[r, 0] * R[0, c] + D[r, 1] * R[1, c]) + D[r, 2] * R[2, c]
        tn[r] = ((D[r, 0] * t[0] + D[r, 1] * t[1]) + D[r, 2] * t[2]) + xi[3 + r]
    return Rn, tn


def optimise(p, q, mu0, iteration_number=64, max_dist=0.025, division_factor=1.4, decrease_mu=1, trace=None):
    """T = (R, t) after iteration_number steps (the normalised target onto the normalised source)."""
    R, t = np.eye(3), np.zeros(3)
    for mu in mu_schedule(mu0, iteration_number, max_dist, division_factor, decrease_mu):
        v, w = system(p, q, R, t, mu)
        A, g = unpack(v)
        xi = solve6(A, g)
        if trace is not None:
            trace.append(dict(mu=mu, A=A, g=g, xi=xi, w=w))
        if np.isfinite(xi).all():
            R, t = step(R, t, xi)
    return R, t


def to_input_frame(R, t, info):
    """The result mapping the source onto the target: (R^T, -(R^T t')) with t' = (-(R mu_t) + scale_global t) +
    mu_s."""
    mt, ms, sg = info["mean_t"], info["mean_s"], info["scale_global"]
    tp = np.empty(3)
    for r in range(3):
        Rm = (R[r, 0] * mt[0] + R[r, 1] * mt[1]) + R[r, 2] * mt[2]
        tp[r] = (-Rm + sg * t[r]) + ms[r]
    Ro = R.T.copy()
    to = np.array([-((Ro[r, 0] * tp[0] + Ro[r, 1] * tp[1]) + Ro[r, 2] * tp[2]) for r in range(3)])
    return Ro, to


def fgr(x, y, corr, division_factor=1.4, use_absolute_scale=0, decrease_mu=1, maximum_correspondence_distance=0.025,
        iteration_number=64):
    """The header's FGR of one problem: dict(R, t, iterations, converged, K) (R, t: the source onto the target)."""
    p, q, info = normalise(x, y, corr, use_absolute_scale)
    if info["K"] < MIN_CORR or iteration_number == 0:
        return dict(R=np.eye(3), t=np.zeros(3), iterations=0, converged=0, info=info)
    R, t = optimise(p, q, info["mu0"], iteration_number, maximum_correspondence_distance, division_factor, decrease_mu)
    Ro, to = to_input_frame(R, t, info)
    return dict(R=Ro, t=to, iterations=iteration_number, converged=1, info=info)
