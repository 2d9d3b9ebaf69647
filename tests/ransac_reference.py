"""Numpy float64 restatement of correspondence RANSAC as include/teaser_b200.h defines it (tzr_ransac_batch, DESIGN.md
§3.21): the draws, the checkers, the Kabsch estimate, the segment-ordered score and the sequential loop with its exit
bound, in the device's order.

The generator runs on Python integers; the Kabsch rotation is tests/rotation_reference.svd_rot, a bit-exact replica
of the device's rotation_from_H; every product and sum follows the header's parentheses; the score's sum of d^2 runs
segment by segment (np.cumsum adds in order).  The only host/device difference is log() in the exit bound (the host
libm against CUDA's, an ulp apart at most), so ransac() reports how far every bound it applied lay from an integer, and
exact drawn counts are only worth asserting where that margin is not tiny.  The evaluation (tzr_icp_batch with
max_iteration = 0) is not restated here.
"""
from __future__ import annotations

import math

import numpy as np

from rotation_reference import svd_rot

SEG = 512
MASK = (1 << 64) - 1


def splitmix64(x):
    x = (x + 0x9E3779B97F4A7C15) & MASK
    x = ((x ^ (x >> 30)) * 0xBF58476D1CE4E5B9) & MASK
    x = ((x ^ (x >> 27)) * 0x94D049BB133111EB) & MASK
    return x ^ (x >> 31)


def draws(seed, n, itr, Kv):
    """The rows of hypothesis itr: mulhi64(splitmix64(seed + n itr + j), Kv) for j < n."""
    return [(splitmix64((seed + n * itr + j) & MASK) * Kv) >> 64 for j in range(n)]


def usable(x, y, corr, xn=None, yn=None):
    """(rows x, rows y, rows of normals or None): the correspondences with both ends finite, in input order, as
    float64 (the float32 inputs read exactly)."""
    x = np.asarray(x, dtype=np.float32).astype(np.float64)
    y = np.asarray(y, dtype=np.float32).astype(np.float64)
    corr = np.asarray(corr, dtype=np.int64).reshape(-1, 2)
    X, Y = x[corr[:, 0]], y[corr[:, 1]]
    ok = np.isfinite(X).all(axis=1) & np.isfinite(Y).all(axis=1)
    N = None
    if xn is not None:
        xn = np.asarray(xn, dtype=np.float32)[:, :3].astype(np.float64)
        yn = np.asarray(yn, dtype=np.float32)[:, :3].astype(np.float64)
        N = (xn[corr[:, 0]][ok], yn[corr[:, 1]][ok])
    return X[ok], Y[ok], N


def _norm(a, b):
    d = [a[0] - b[0], a[1] - b[1], a[2] - b[2]]
    return math.sqrt((d[0] * d[0] + d[1] * d[1]) + d[2] * d[2])


def edge_ok(P, Q, s):
    """Edge-length checker: fails when d_x < d_y s or d_y < d_x s for some pair i < j."""
    n = len(P)
    for i in range(n):
        for j in range(i + 1, n):
            ds, dt = _norm(P[i], P[j]), _norm(Q[i], Q[j])
            if ds < dt * s or dt < ds * s:
                return False
    return True


def kabsch(P, Q):
    """(R, t): means in draw order from 0 divided by n, H(r, c) summed in draw order from 0, R = svd_rot(H),
    t(r) = mu_q(r) - ((R(r,0) mu_p0 + R(r,1) mu_p1) + R(r,2) mu_p2)."""
    n = len(P)
    mp, mq = [0.0, 0.0, 0.0], [0.0, 0.0, 0.0]
    for k in range(n):
        for d in range(3):
            mp[d] = mp[d] + float(P[k][d])
            mq[d] = mq[d] + float(Q[k][d])
    mp = [v / float(n) for v in mp]
    mq = [v / float(n) for v in mq]
    H = np.zeros((3, 3))
    for k in range(n):
        u = [float(P[k][d]) - mp[d] for d in range(3)]
        w = [float(Q[k][d]) - mq[d] for d in range(3)]
        for c in range(3):
            for r in range(3):
                H[r, c] = H[r, c] + u[r] * w[c]
    R = svd_rot(H)
    t = np.array([mq[r] - ((R[r, 0] * mp[0] + R[r, 1] * mp[1]) + R[r, 2] * mp[2]) for r in range(3)])
    return R, t


def d2_rows(R, t, X, Y):
    """d^2 of every row: each component ((R(r,0) x0 + R(r,1) x1) + R(r,2) x2) + t(r) - y(r), then (e0 e0 + e1 e1) + e2 e2."""
    e = [((R[r, 0] * X[:, 0] + R[r, 1] * X[:, 1]) + R[r, 2] * X[:, 2]) + t[r] - Y[:, r] for r in range(3)]
    return (e[0] * e[0] + e[1] * e[1]) + e[2] * e[2]


def distance_ok(R, t, P, Q, thr):
    return not any(math.sqrt(v) > thr for v in d2_rows(R, t, np.asarray(P), np.asarray(Q)))


def normal_ok(R, NP, NQ, cos_thr):
    """Normal checker: fails when (n_y0 m0 + n_y1 m1) + n_y2 m2 < cos_thr, m = R n_x (a NaN never fails)."""
    for a, b in zip(NP, NQ):
        m = [(R[r, 0] * a[0] + R[r, 1] * a[1]) + R[r, 2] * a[2] for r in range(3)]
        if (b[0] * m[0] + b[1] * m[1]) + b[2] * m[2] < cos_thr:
            return False
    return True


def score(R, t, X, Y, r2):
    """(count, sum d^2, fitness, rmse) over the usable rows: inliers d^2 < r2, each segment of SEG rows summed in
    ascending order from 0, the segment sums added in ascending order from 0."""
    d2 = d2_rows(R, t, X, Y)
    inl = d2 < r2
    count = int(inl.sum())
    total = 0.0
    for s0 in range(0, len(d2), SEG):
        seg = np.where(inl[s0:s0 + SEG], d2[s0:s0 + SEG], 0.0)
        part = float(np.cumsum(np.concatenate([[0.0], seg]))[-1])
        total = total + part
    fit = count / len(X) if count else 0.0
    rmse = math.sqrt(total / count) if count else 0.0
    return count, total, fit, rmse


def better(fa, ra, fb, rb):
    return fa > fb or (fa == fb and ra < rb)


def bound(f, n, confidence):
    """(bound, raw): ceil(log(1 - confidence) / log(1 - f^n)) with f^n = ((f f) f) ...; +inf when that is NaN or -inf.
    raw is the quotient before ceil (for the margin)."""
    fn = f
    for _ in range(1, n):
        fn = fn * f
    num = math.log(1.0 - confidence) if confidence < 1.0 else -math.inf
    den = math.log(1.0 - fn) if fn < 1.0 else -math.inf
    with np.errstate(all="ignore"):
        q = float(np.float64(num) / np.float64(den))
    b = math.ceil(q) if math.isfinite(q) else q
    if not (b >= 0.0):  # NaN or -inf: no bound
        return math.inf, q
    return b, q


def hypothesis(X, Y, N, itr, seed, n, edge=None, dist=None, cos_normal=None):
    """(passed, R, t) of hypothesis itr."""
    rows = draws(seed, n, itr, len(X))
    P, Q = X[rows], Y[rows]
    if edge is not None and not edge_ok(P, Q, edge):
        return False, None, None
    R, t = kabsch(P, Q)
    if dist is not None and not distance_ok(R, t, P, Q, dist):
        return False, R, t
    if cos_normal is not None and not normal_ok(R, N[0][rows], N[1][rows], cos_normal):
        return False, R, t
    return True, R, t


def ransac(x, y, corr, r, seed=0, ransac_n=3, max_iteration=100000, confidence=0.999, edge=None, dist=None,
           normal_angle=None, xn=None, yn=None):
    """The sequential loop.  edge / dist / normal_angle: the checkers' thresholds (None: off).  Returns a dict: R, t
    (the winner's, or the identity), drawn, passed, winner (-1: none), inliers, rmse, usable, converged, and margin:
    the smallest distance of a raw bound that lowered exit from its nearest integer (inf when none did)."""
    X, Y, N = usable(x, y, corr, xn, yn)
    Kv = len(X)
    r2 = r * r
    cos_normal = None if normal_angle is None else math.cos(normal_angle)
    out = dict(R=np.eye(3), t=np.zeros(3), drawn=0, passed=0, winner=-1, inliers=0, rmse=0.0, fitness=0.0, usable=Kv,
               converged=0, margin=math.inf)
    if Kv < ransac_n or max_iteration == 0:
        return out
    bf, brm, exit_ = 0.0, 0.0, float(max_iteration)
    itr = 0
    while itr < max_iteration and itr < exit_:
        ok, R, t = hypothesis(X, Y, N, itr, seed, ransac_n, edge, dist, cos_normal)
        if ok:
            out["passed"] += 1
            cnt, _, f, rm = score(R, t, X, Y, r2)
            if better(f, rm, bf, brm):
                bf, brm = f, rm
                b, q = bound(f, ransac_n, confidence)
                out.update(R=R, t=t, winner=itr, inliers=cnt, rmse=rm, fitness=f)
                if b < exit_:
                    exit_ = b
                    if math.isfinite(q):
                        out["margin"] = min(out["margin"], abs(q - round(q)))
        itr += 1
    out["drawn"] = itr
    out["converged"] = int(itr < max_iteration)
    return out


def literal_ransac(x, y, corr, r, seed=0, ransac_n=3, max_iteration=100, confidence=0.999):
    """An unoptimised transcription of the header's loop with no checkers (every hypothesis scored row by row, the
    sums in plain loops): the premise check of ransac()."""
    X, Y, _ = usable(x, y, corr)
    Kv = len(X)
    best = None
    if Kv < ransac_n or max_iteration == 0:
        return dict(drawn=0, winner=-1)
    exit_ = max_iteration
    itr = 0
    bf, brm = 0.0, 0.0
    while itr < max_iteration and itr < exit_:
        rows = draws(seed, ransac_n, itr, Kv)
        R, t = kabsch(X[rows], Y[rows])
        count, total, seg = 0, 0.0, 0.0
        for k in range(Kv):
            if k % SEG == 0 and k:
                total, seg = total + seg, 0.0
            e = [((R[q, 0] * X[k, 0] + R[q, 1] * X[k, 1]) + R[q, 2] * X[k, 2]) + t[q] - Y[k, q] for q in range(3)]
            d2 = (e[0] * e[0] + e[1] * e[1]) + e[2] * e[2]
            if d2 < r * r:
                count += 1
                seg = seg + d2
        total = total + seg
        f = count / Kv if count else 0.0
        rm = math.sqrt(total / count) if count else 0.0
        if better(f, rm, bf, brm):
            bf, brm, best = f, rm, (itr, R, t, count)
            b, _ = bound(f, ransac_n, confidence)
            exit_ = min(exit_, b)
        itr += 1
    return dict(drawn=itr, winner=-1 if best is None else best[0], R=None if best is None else best[1],
                t=None if best is None else best[2], inliers=0 if best is None else best[3], rmse=brm)
