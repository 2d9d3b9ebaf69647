"""One ICP step of include/teaser_b200.h in exact arithmetic, for point-to-point, point-to-plane, generalized ICP and
the robust kernels of both Gauss-Newton systems.

The numpy restatements (tests/icp_reference.py and the three that build on it) follow the header's formulas in float64,
so a wrong formula copied into both sides agrees with itself.  This module computes the operation the header defines,
from the float inputs, without rounding:

  - the transform p = s (R x) + t, the centroids, every sum (the covariance H, the 27 Gauss-Newton sums) and the
    truncated, diagonally pivoted LDL^T of the 6 x 6 solve are fractions.Fraction.  The pivot rule (the largest remaining
    diagonal, the lowest index on ties) and the truncation (stop unless that diagonal is > tol) are applied to the
    exact values; tol is the header's float64 product fl(1e-10 max_k A_kk), so that a diagonal equal to it is decided
    as the device decides it;
  - point-to-point's rotation is found without an SVD, by Horn's quaternion: the top eigenvector of the symmetric 4 x 4
    matrix N(H) at PREC bits;
  - Rz(x2) Ry(x1) Rx(x0) uses mpmath's sin and cos at PREC bits;
  - generalized ICP's A = M^-1 is the exact inverse of the exact M = s^2 C(R m) + C(n), not the adjugate in floats;
    the robust GICP's W = M^-1/2 comes from mpmath's eigendecomposition of M at PREC bits.

Quotients by a per-correspondence value (the entries of M^-1, the robust weights) would give every term of a sum its
own denominator and make the sums' size grow with the count.  Those values alone are rounded to PREC = 256 bits (a
dyadic Fraction) before they enter the sums: a relative change of 2^-256, about 200 bits below float64's unit roundoff,
so "exact" means exact to far below anything the device can resolve.

Each step returns R, t (float64 of the exact values), the exact A, g and x (Fractions; None for point-to-point), the
rank the truncation reached, and a condition measure for a tolerance: for Kabsch the gap sigma_2 + sigma_3 of H (the
rotation's sensitivity to a perturbation dH is |dH| / (sigma_2 + sigma_3)), for Gauss-Newton the extreme eigenvalues
of A restricted to the pivoted block.
"""
from __future__ import annotations

from fractions import Fraction as F

import mpmath
import numpy as np

PREC = 256
TOL_FACTOR = 1e-10  # the double the device multiplies by
LOSSES = {"l2": 0, "l1": 1, "huber": 2, "cauchy": 3, "gm": 4, "tukey": 5}


def _ctx():
    mpmath.mp.prec = PREC
    return mpmath.mp


def _mpf(q):
    return mpmath.mpf(q.numerator) / q.denominator


def _frac(v):
    """An mpf as the Fraction of its exact value."""
    sign, man, exp, _ = mpmath.mpf(v)._mpf_
    if not man:
        return F(0)
    return (-1) ** sign * F(int(man)) * (F(2) ** int(exp))


def rounded(q):
    """q (a Fraction) rounded to PREC bits, as a Fraction."""
    _ctx()
    return _frac(_mpf(q))


def exact_points(a):
    """Rows of float values (float32 or float64) as lists of exact Fractions."""
    return [[F(float(v)) for v in row] for row in np.asarray(a)]


def transform(xs, s, R, t):
    """p = s (R x) + t exactly, for rows x of Fractions; s, R, t: floats (their exact values)."""
    s, t = F(float(s)), [F(float(v)) for v in np.asarray(t).reshape(3)]
    R = [[F(float(R[r][c])) for c in range(3)] for r in range(3)]
    return [[s * (R[r][0] * x[0] + R[r][1] * x[1] + R[r][2] * x[2]) + t[r] for r in range(3)] for x in xs]


def _mean(rows):
    n = len(rows)
    return [sum((p[k] for p in rows), F(0)) / n for k in range(3)]


def _cross(a, b):
    return [a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]]


def _matvec(M, v):
    return [sum((M[r][c] * v[c] for c in range(len(v))), F(0)) for r in range(len(M))]


# ---- the truncated, pivoted LDL^T ---------------------------------------------------------------------------------

def solve6(A, g):
    """x with A x = -g by the header's truncated LDL^T with diagonal pivoting, on exact values (Fractions).  Returns
    (x, rank, pivots)."""
    S = [[F(A[i][j]) for j in range(6)] for i in range(6)]
    amax = max(S[i][i] for i in range(6))
    tol = F(TOL_FACTOR * float(amax))  # fl(1e-10 amax)
    used, piv, d = [False] * 6, [], []
    L = [[F(0)] * 6 for _ in range(6)]
    for s in range(6):
        best = -1
        for i in range(6):
            if not used[i] and (best < 0 or S[i][i] > S[best][best]):
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
    y = [F(0)] * rank
    for s in range(rank):
        y[s] = -F(g[piv[s]]) - sum((L[piv[s]][q] * y[q] for q in range(s)), F(0))
    for s in range(rank):
        y[s] = y[s] / d[s]
    for s in range(rank - 1, -1, -1):
        y[s] = y[s] - sum((L[piv[q]][s] * y[q] for q in range(s + 1, rank)), F(0))
    x = [F(0)] * 6
    for s in range(rank):
        x[piv[s]] = y[s]
    return x, rank, piv


def block_eigenvalues(A, piv):
    """(smallest, largest) eigenvalue of A restricted to the rows and columns piv, at PREC bits; (inf, 0) for none."""
    if not piv:
        return float("inf"), 0.0
    mp = _ctx()
    E = mp.eigsy(mp.matrix([[_mpf(F(A[i][j])) for j in piv] for i in piv]), eigvals_only=True)
    ev = sorted(float(e) for e in E)
    return ev[0], ev[-1]


def euler(x0, x1, x2):
    """Rz(x2) Ry(x1) Rx(x0) of exact angles, as a PREC-bit mpmath matrix."""
    mp = _ctx()
    a, b, c = _mpf(x0), _mpf(x1), _mpf(x2)
    Rx = mp.matrix([[1, 0, 0], [0, mp.cos(a), -mp.sin(a)], [0, mp.sin(a), mp.cos(a)]])
    Ry = mp.matrix([[mp.cos(b), 0, mp.sin(b)], [0, 1, 0], [-mp.sin(b), 0, mp.cos(b)]])
    Rz = mp.matrix([[mp.cos(c), -mp.sin(c), 0], [mp.sin(c), mp.cos(c), 0], [0, 0, 1]])
    return Rz * Ry * Rx


def _compose(Ru, tu, R, t):
    """R <- Ru R, t <- Ru t + tu (Ru: mpmath matrix, tu: mpf list), as float64 arrays of the exact values."""
    mp = _ctx()
    R0 = mp.matrix([[mpmath.mpf(float(R[r][c])) for c in range(3)] for r in range(3)])
    t0 = mp.matrix([mpmath.mpf(float(v)) for v in np.asarray(t).reshape(3)])
    Rn, tn = Ru * R0, Ru * t0
    return (np.array([[float(Rn[r, c]) for c in range(3)] for r in range(3)]),
            np.array([float(tn[r] + tu[r]) for r in range(3)]))


# ---- point-to-point ------------------------------------------------------------------------------------------------

def horn_rotation(H):
    """The rotation R maximising sum w . R u for H = sum u w^T (Fractions), from the top eigenvector of Horn's N(H)."""
    mp = _ctx()
    S = [[_mpf(H[r][c]) for c in range(3)] for r in range(3)]
    (xx, xy, xz), (yx, yy, yz), (zx, zy, zz) = S
    N = mp.matrix([[xx + yy + zz, yz - zy, zx - xz, xy - yx],
                   [yz - zy, xx - yy - zz, xy + yx, zx + xz],
                   [zx - xz, xy + yx, -xx + yy - zz, yz + zy],
                   [xy - yx, zx + xz, yz + zy, -xx - yy + zz]])
    E, Q = mp.eigsy(N)
    k = max(range(4), key=lambda i: E[i])
    q0, qx, qy, qz = (Q[i, k] for i in range(4))
    return mp.matrix([[q0 * q0 + qx * qx - qy * qy - qz * qz, 2 * (qx * qy - q0 * qz), 2 * (qx * qz + q0 * qy)],
                      [2 * (qx * qy + q0 * qz), q0 * q0 - qx * qx + qy * qy - qz * qz, 2 * (qy * qz - q0 * qx)],
                      [2 * (qx * qz - q0 * qy), 2 * (qy * qz + q0 * qx), q0 * q0 - qx * qx - qy * qy + qz * qz]])


def step_point(x, y, corr, s, R, t):
    """One point-to-point step from the correspondences corr ((m,2) rows (source, target)) at the seed (s, R, t):
    centred Kabsch for 3 or more, the translation of the centroids for 1 or 2, the identity for none."""
    mp = _ctx()
    corr = np.asarray(corr, dtype=np.int64).reshape(-1, 2)
    out = dict(A=None, g=None, x=None, rank=None, gap=None, H=None)
    if len(corr) == 0:
        R1, t1 = _compose(mp.eye(3), [mpmath.mpf(0)] * 3, R, t)
        return dict(out, R=R1, t=t1, count=0)
    P = transform(exact_points(np.asarray(x)[corr[:, 0]]), s, R, t)
    Q = exact_points(np.asarray(y)[corr[:, 1]])
    mp_, mq = _mean(P), _mean(Q)
    if len(corr) < 3:
        R1, t1 = _compose(mp.eye(3), [_mpf(mq[k] - mp_[k]) for k in range(3)], R, t)
        return dict(out, R=R1, t=t1, count=len(corr), mu_p=mp_, mu_q=mq)
    U = [[p[k] - mp_[k] for k in range(3)] for p in P]
    W = [[q[k] - mq[k] for k in range(3)] for q in Q]
    H = [[sum((u[r] * w[c] for u, w in zip(U, W)), F(0)) for c in range(3)] for r in range(3)]
    Ru = horn_rotation(H)
    tu = [_mpf(mq[r]) - sum(Ru[r, c] * _mpf(mp_[c]) for c in range(3)) for r in range(3)]
    sv = sorted((float(v) for v in mp.svd_r(mp.matrix([[_mpf(H[r][c]) for c in range(3)] for r in range(3)]),
                                               compute_uv=False)), reverse=True)
    R1, t1 = _compose(Ru, tu, R, t)
    return dict(out, R=R1, t=t1, count=len(corr), H=H, gap=sv[1] + sv[2], sigma=sv, mu_p=mp_, mu_q=mq,
                Ru=np.array([[float(Ru[r, c]) for c in range(3)] for r in range(3)]))


# ---- Gauss-Newton systems ------------------------------------------------------------------------------------------

def weight(loss, k, r):
    """The header's weight rho'(r) / r of kernel `loss` (a LOSSES value) with parameter k at the exact residual r (a
    Fraction), rounded to PREC bits; None where it is not finite (L1 at r = 0)."""
    e, k = abs(r), F(float(k))
    if loss == LOSSES["l2"]:
        return F(1)
    if loss == LOSSES["l1"]:
        return None if e == 0 else rounded(1 / e)
    if loss == LOSSES["huber"]:
        return rounded(k / max(e, k))
    if loss == LOSSES["cauchy"]:
        q = e / k
        return rounded(1 / (1 + q * q))
    if loss == LOSSES["gm"]:
        tt = k + e * e
        return rounded(k / (tt * tt))
    if loss == LOSSES["tukey"]:
        if e > k:
            return F(0)
        q = e / k
        return rounded((1 - q * q) ** 2)
    raise ValueError(f"unknown loss {loss}")


def _finite(v):
    return bool(np.isfinite(np.asarray(v, dtype=np.float64)).all())


def _gn_finish(A, g, c, R, t, count, extra):
    x, rank, piv = solve6(A, g)
    Ru = euler(*x[:3])
    tu = [_mpf(c[r] + x[3 + r]) - sum(Ru[r, q] * _mpf(c[q]) for q in range(3)) for r in range(3)]
    R1, t1 = _compose(Ru, tu, R, t)
    lo, hi = block_eigenvalues(A, piv)
    return dict(extra, R=R1, t=t1, A=A, g=g, x=x, rank=rank, piv=piv, lam_min=lo, lam_max=hi, count=count, c=c,
                Ru=np.array([[float(Ru[r, q]) for q in range(3)] for r in range(3)]))


def _identity(R, t, count):
    mp = _ctx()
    R1, t1 = _compose(mp.eye(3), [mpmath.mpf(0)] * 3, R, t)
    return dict(R=R1, t=t1, A=None, g=None, x=None, rank=0, piv=[], count=count)


def _accumulate(A, g, Jrows, Acov, d, w=F(1)):
    """A += w J^T Acov J, g += w J^T Acov d for the 3 x 6 J given as rows (or, with Acov None, the 1 x 6 row Jrows[0]
    and the scalar residual d: A += w J J^T, g += w J d)."""
    if Acov is None:
        J = Jrows[0]
        wJ = [w * v for v in J]
        for a in range(6):
            for b in range(a, 6):
                A[a][b] += wJ[a] * J[b]
            g[a] += wJ[a] * d
        return
    AJ = [[sum((Acov[r][q] * Jrows[q][col] for q in range(3)), F(0)) for col in range(6)] for r in range(3)]
    Ad = _matvec(Acov, d)
    for a in range(6):
        for b in range(a, 6):
            A[a][b] += sum((Jrows[q][a] * AJ[q][b] for q in range(3)), F(0))
        g[a] += sum((Jrows[q][a] * Ad[q] for q in range(3)), F(0))


def _mirror(A):
    for a in range(6):
        for b in range(a):
            A[a][b] = A[b][a]
    return A


def step_plane(x, y, normals, corr, s, R, t, loss=None, k=1.0):
    """One point-to-plane step (loss: a LOSSES value for the robust system, None or "l2" for the plain one): the exact
    A = sum w J J^T and g = sum w J r about c = mu_p of all correspondences, J = ((p - c) x n, n), r = (p - q) . n, over
    the correspondences whose normal is finite (and weight finite); the truncated solve; Rz Ry Rx."""
    loss = LOSSES.get(loss, loss) if loss is not None else None
    corr = np.asarray(corr, dtype=np.int64).reshape(-1, 2)
    if len(corr) == 0:
        return _identity(R, t, 0)
    P = transform(exact_points(np.asarray(x)[corr[:, 0]]), s, R, t)
    c = _mean(P)
    Nf = np.asarray(normals, dtype=np.float32)[:, :3][corr[:, 1]]
    Qf = np.asarray(y)[corr[:, 1]]
    A = [[F(0)] * 6 for _ in range(6)]
    g = [F(0)] * 6
    used = 0
    for p, qf, nf in zip(P, Qf, Nf):
        if not _finite(nf):
            continue
        n, q = exact_points([nf])[0], exact_points([qf])[0]
        u = [p[k2] - c[k2] for k2 in range(3)]
        J = _cross(u, n) + n
        r = sum(((p[k2] - q[k2]) * n[k2] for k2 in range(3)), F(0))
        w = F(1) if loss in (None, LOSSES["l2"]) else weight(loss, k, r)
        if w is None:
            continue
        _accumulate(A, g, [J], None, r, w)
        used += 1
    return _gn_finish(_mirror(A), g, c, R, t, len(corr), dict(used=used))


def covariance(v, epsilon):
    """C(v) = I - (1 - epsilon) v v^T / (v . v) exactly (v: Fractions)."""
    e = F(float(epsilon))
    kk = (1 - e) / sum((a * a for a in v), F(0))
    return [[(F(1) if a == b else F(0)) - kk * v[a] * v[b] for b in range(3)] for a in range(3)]


def inverse3(M):
    """The exact inverse of a 3 x 3 Fraction matrix and its determinant (None when singular)."""
    c = [[M[(r + 1) % 3][(q + 1) % 3] * M[(r + 2) % 3][(q + 2) % 3] - M[(r + 1) % 3][(q + 2) % 3] *
          M[(r + 2) % 3][(q + 1) % 3] for q in range(3)] for r in range(3)]
    det = sum((M[0][q] * c[0][q] for q in range(3)), F(0))
    if det == 0:
        return None, det
    return [[c[q][r] / det for q in range(3)] for r in range(3)], det


def whitening(M):
    """W = M^-1/2 (PREC-bit mpmath matrix) from the eigendecomposition of the exact M, and the eigenvalues."""
    mp = _ctx()
    E, V = mp.eigsy(mp.matrix([[_mpf(M[r][q]) for q in range(3)] for r in range(3)]))
    if min(E[i] for i in range(3)) <= 0:
        return None, [float(E[i]) for i in range(3)]
    D = mp.diag([1 / mp.sqrt(E[i]) for i in range(3)])
    return V * D * V.T, [float(E[i]) for i in range(3)]


def step_generalized(x, y, src_normals, dst_normals, corr, s, R, t, epsilon, loss=None, k=1.0):
    """One generalized-ICP step (loss as step_plane's): per correspondence with finite, non-zero normals m and n,
    M = s^2 C(R m) + C(n) exactly; A = M^-1 (exact, rounded to PREC bits), or for a robust loss A~ = W diag(w) W with
    W = M^-1/2 and w_k the weight of r_k = W_k . d; the sums J^T A J and J^T A d with J = [e_k x u, I], u = p - c,
    d = p - q; the truncated solve; Rz Ry Rx.  Also returns kappa, the largest condition number of any M used."""
    mp = _ctx()
    loss = LOSSES.get(loss, loss) if loss is not None else None
    corr = np.asarray(corr, dtype=np.int64).reshape(-1, 2)
    if len(corr) == 0:
        return _identity(R, t, 0)
    P = transform(exact_points(np.asarray(x)[corr[:, 0]]), s, R, t)
    c = _mean(P)
    Ms = np.asarray(src_normals, dtype=np.float32)[:, :3][corr[:, 0]]
    Nt = np.asarray(dst_normals, dtype=np.float32)[:, :3][corr[:, 1]]
    Qf = np.asarray(y)[corr[:, 1]]
    Rf = [[F(float(R[r][q])) for q in range(3)] for r in range(3)]
    s2 = F(float(s)) ** 2
    A = [[F(0)] * 6 for _ in range(6)]
    g = [F(0)] * 6
    used, kappa = 0, 1.0
    for p, qf, mf, nf in zip(P, Qf, Ms, Nt):
        if not (_finite(mf) and _finite(nf)):
            continue
        m0, n, q = exact_points([mf])[0], exact_points([nf])[0], exact_points([qf])[0]
        if not any(m0) or not any(n):
            continue
        m = _matvec(Rf, m0)
        Cm, Cn = covariance(m, epsilon), covariance(n, epsilon)
        M = [[s2 * Cm[a][b] + Cn[a][b] for b in range(3)] for a in range(3)]
        d = [p[a] - q[a] for a in range(3)]
        if loss in (None, LOSSES["l2"]):
            Ainv, det = inverse3(M)
            if Ainv is None or det <= 0:
                continue
            Acov = [[rounded(Ainv[a][b]) for b in range(3)] for a in range(3)]
        else:
            Wm, sig = whitening(M)
            if Wm is None:
                continue
            dm = [_mpf(v) for v in d]
            w = []
            for kk in range(3):
                rk = sum(Wm[kk, b] * dm[b] for b in range(3))
                wk = weight(loss, k, _frac(rk))
                if wk is None:
                    break
                w.append(_mpf(wk))
            if len(w) < 3:
                continue
            Acov = [[_frac(sum(w[kk] * Wm[kk, a] * Wm[kk, b] for kk in range(3))) for b in range(3)] for a in range(3)]
        E = np.linalg.eigvalsh(np.array([[float(M[a][b]) for b in range(3)] for a in range(3)]))
        kappa = max(kappa, float(E[-1] / E[0]))  # a tolerance's measure: float64 is plenty
        u = [p[a] - c[a] for a in range(3)]
        # J = [e_k x u (k = 0..2), I]: row r of e_k x u is (e_k x u)_r
        Jrows = [[_cross([F(int(kk == 0)), F(int(kk == 1)), F(int(kk == 2))], u)[r] for kk in range(3)] +
                 [F(int(r == q2)) for q2 in range(3)] for r in range(3)]
        _accumulate(A, g, Jrows, Acov, d)
        used += 1
    return _gn_finish(_mirror(A), g, c, R, t, len(corr), dict(used=used, kappa=kappa))


def step(method, x, y, corr, s, R, t, src_normals=None, dst_normals=None, epsilon=1e-3, loss=None, k=1.0):
    """step_point, step_plane or step_generalized by name ("point", "plane", "generalized")."""
    if method == "point":
        return step_point(x, y, corr, s, R, t)
    if method == "plane":
        return step_plane(x, y, dst_normals, corr, s, R, t, loss, k)
    return step_generalized(x, y, src_normals, dst_normals, corr, s, R, t, epsilon, loss, k)
