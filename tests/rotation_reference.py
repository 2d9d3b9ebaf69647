"""Plain reference of the rotation stage (csrc/rot_trans.cu) as the device runs it, and an exact Procrustes reference.

Independent of the CPU oracle.  The kernel is compiled with -fmad=false and its rotation arithmetic is IEEE + - * /
sqrt only, so a float64 replay in the same operation order must equal it bit for bit:

svd_rot(H)     svd3 (two-sided Jacobi) + the reflection fix, R = V U^T, for H = sum_k x_k y_k^T (R maps x to y).
yaw_rot(H)     the planar closed form of rotation_step (Quatro): the yaw maximising tr(R H) over the top-left 2x2 block.
               Both first bring H to [1/2, 1) by a power of two when its largest |entry| lies outside
               [2^-400, 2^400] (normalise=False replays the unscaled algorithm).
Tims           a TIM set and the kernel's thread map: CHAIN puts TIM k on thread k mod 128; COMPLETE walks i in order and
               gives pair (i, j) to thread (j - i - 1) mod 128 (for_each_tim).  block_sum() replays block_sum<K> with
               128 threads: per-thread sequential sums from 0.0, the xor butterfly inside each warp, the four warp
               partials in order.
gnc_tls(), fgr(), quatro()
               the loops of gnc_tls_block / fgr_block; each returns R, cost, iterations, weights and mask.
chain_tims(), complete_tims(), rotation_noise_bound()
               the solve path's TIMs from the sorted clique and the scale: dst differences times (1 / scale), the
               rotation noise bound noise_bound * (2 / scale).
procrustes_exact(H), yaw_exact(H)
               the maximiser of tr(R H) over SO(3) (Horn's quaternion matrix, mpmath at 60 digits) and over planar
               rotations (atan2); with the spectral gap that says how well R is determined.
"""
from __future__ import annotations

import math

import numpy as np

EPS = 2.220446049250313e-16
TINY = 2.2250738585072014e-308
THREADS = 128
WARPS = THREADS // 32
SCALE_LO, SCALE_HI = 2.0 ** -400, 2.0 ** 400


# ------------------------------------------------------------------------------------------------ 3x3 SVD rotation
def _normalised(vals, normalise=True):
    """The values times the power of two that brings the largest |value| into [1/2, 1), if that lies outside
    [2^-400, 2^400]; unchanged otherwise (and for a zero or non-finite maximum)."""
    vals = [float(v) for v in vals]
    mx = max(abs(v) for v in vals)
    if normalise and math.isfinite(mx) and mx > 0.0 and (mx < SCALE_LO or mx > SCALE_HI):
        e = math.frexp(mx)[1]
        vals = [math.ldexp(v, -e) for v in vals]
    return vals


def _det(m):
    return (m[0][0] * (m[1][1] * m[2][2] - m[1][2] * m[2][1]) - m[0][1] * (m[1][0] * m[2][2] - m[1][2] * m[2][0]) +
            m[0][2] * (m[1][0] * m[2][1] - m[1][1] * m[2][0]))


def _rot_rows(A, p, q, c, s):
    for col in range(3):
        xp, xq = A[p][col], A[q][col]
        A[p][col] = c * xp + s * xq
        A[q][col] = c * xq - s * xp


def _rot_cols(A, p, q, c, s):
    for row in range(3):
        xp, xq = A[row][p], A[row][q]
        A[row][p] = c * xp - s * xq
        A[row][q] = s * xp + c * xq


def svd3(H):
    """H = U diag(S) V^T by the kernel's two-sided Jacobi; returns (U, S, V, sweeps) as nested lists."""
    A = [[float(H[r][c]) for c in range(3)] for r in range(3)]
    U = [[1.0 if r == c else 0.0 for c in range(3)] for r in range(3)]
    V = [row[:] for row in U]
    max_diag = max(abs(A[0][0]), max(abs(A[1][1]), abs(A[2][2])))
    sweeps = 0
    for sweep in range(64):
        sweeps = sweep + 1
        finished = True
        for p in (1, 2):
            for q in range(p):
                thr = max(TINY, 2.0 * EPS * max_diag)
                if abs(A[p][q]) > thr or abs(A[q][p]) > thr:
                    finished = False
                    m00, m01, m10, m11 = A[p][p], A[p][q], A[q][p], A[q][q]
                    t, d = m00 + m11, m10 - m01
                    if abs(d) < TINY:
                        c1, s1 = 1.0, 0.0
                    else:
                        u = t / d
                        h = math.sqrt(1.0 + u * u)
                        s1 = 1.0 / h
                        c1 = u / h
                    n00 = c1 * m00 + s1 * m10
                    n01 = c1 * m01 + s1 * m11
                    n11 = c1 * m11 - s1 * m01
                    if 2.0 * abs(n01) < TINY:
                        c2, s2 = 1.0, 0.0
                    else:
                        tau = (n00 - n11) / (2.0 * n01)
                        w = math.sqrt(tau * tau + 1.0)
                        tt = -1.0 / (tau + w) if tau >= 0.0 else 1.0 / (w - tau)
                        c2 = 1.0 / math.sqrt(tt * tt + 1.0)
                        s2 = tt * c2
                    cl = c2 * c1 + s2 * s1
                    sl = c2 * s1 - s2 * c1
                    _rot_rows(A, p, q, cl, sl)
                    _rot_cols(U, p, q, cl, -sl)
                    _rot_cols(A, p, q, c2, s2)
                    _rot_cols(V, p, q, c2, s2)
                    max_diag = max(max_diag, max(abs(A[p][p]), abs(A[q][q])))
        if finished:
            break
    S = [0.0] * 3
    for i in range(3):
        a = A[i][i]
        S[i] = abs(a)
        if a < 0.0:
            for r in range(3):
                U[r][i] = -U[r][i]
    for i in range(3):
        pos = i
        for k in range(i + 1, 3):
            if S[k] > S[pos]:
                pos = k
        if pos != i:
            S[i], S[pos] = S[pos], S[i]
            for r in range(3):
                U[r][i], U[r][pos] = U[r][pos], U[r][i]
                V[r][i], V[r][pos] = V[r][pos], V[r][i]
    return U, S, V, sweeps


def svd_rot(H, normalise=True):
    """rotation_from_H: the proper rotation R = V U^T (reflection fix on V's last column) as a (3, 3) array."""
    H = np.asarray(H, dtype=np.float64)
    h = _normalised(H.ravel(), normalise)
    U, _, V, _ = svd3([h[0:3], h[3:6], h[6:9]])
    if _det(U) * _det(V) < 0.0:
        for r in range(3):
            V[r][2] = -V[r][2]
    R = np.empty((3, 3))
    for r in range(3):
        for c in range(3):
            R[r, c] = V[r][0] * U[c][0] + V[r][1] * U[c][1] + V[r][2] * U[c][2]
    return R


def yaw_rot(H, normalise=True):
    """The planar branch of rotation_step: R = [c -s; s c] (z row and column identity) with (c, s) ~ (h00 + h11,
    h01 - h10); the identity when that vector is zero."""
    H = np.asarray(H, dtype=np.float64)
    h00, h10, h01, h11 = _normalised((H[0, 0], H[1, 0], H[0, 1], H[1, 1]), normalise)
    ca, sb = h00 + h11, h01 - h10
    nrm = math.sqrt(ca * ca + sb * sb)
    R = np.eye(3)
    if nrm > 0.0:
        c, s = ca / nrm, sb / nrm
        R[0, 0], R[0, 1], R[1, 0], R[1, 1] = c, -s, s, c
    return R


# ------------------------------------------------------------------------------------------------ TIM sets + sums
class Tims:
    """x, y: (count, 3) TIMs; lanes: (positions, 128) TIM index held by each thread at each step, -1 where idle."""

    def __init__(self, x, y, lanes):
        self.x = np.ascontiguousarray(x, dtype=np.float64)
        self.y = np.ascontiguousarray(y, dtype=np.float64)
        self.lanes = lanes
        self.count = self.x.shape[0]

    def block_sum(self, v):
        """block_sum<K> of per-TIM values v (count,) or (count, K) -> float or (K,)."""
        v = np.asarray(v, dtype=np.float64)
        one = v.ndim == 1
        v = v.reshape(self.count, -1)
        pad = np.concatenate([v, np.zeros((1, v.shape[1]))])  # index -1: +0.0 leaves a sum started at +0.0 unchanged
        g = pad[self.lanes]  # (positions, 128, K)
        acc = np.zeros((THREADS, v.shape[1]))
        for p in range(g.shape[0]):
            acc = acc + g[p]
        acc = acc.reshape(WARPS, 32, -1)
        lane = np.arange(32)
        for o in (16, 8, 4, 2, 1):
            acc = acc + acc[:, lane ^ o]
        s = np.zeros(v.shape[1])
        for q in range(WARPS):
            s = s + acc[q, 0]
        return float(s[0]) if one else s

    def block_max(self, v, init=0.0):
        v = np.asarray(v, dtype=np.float64)
        return max(init, float(v.max())) if v.size else init


def chain_lanes(count):
    k = np.arange(-(-count // THREADS) * THREADS)
    k[k >= count] = -1
    return k.reshape(-1, THREADS)


def complete_lanes(m):
    rows = []
    for i in range(m - 1):
        base = i * m - i * (i + 1) // 2 - i - 1
        j = np.arange(i + 1, m)
        k = base + j
        n = -(-k.size // THREADS) * THREADS
        pad = np.full(n, -1, dtype=np.int64)
        pad[:k.size] = k
        rows.append(pad.reshape(-1, THREADS))
    return np.concatenate(rows) if rows else np.zeros((0, THREADS), dtype=np.int64)


def plain_tims(x, y):
    """TIMs handed to tzr_rotation_solve (CHAIN map, as given)."""
    x = np.asarray(x, dtype=np.float64).reshape(-1, 3)
    return Tims(x, np.asarray(y, dtype=np.float64).reshape(-1, 3), chain_lanes(x.shape[0]))


def chain_tims(src, dst, clique, scale):
    """CHAIN TIMs of the sorted clique: leaf = next clique point (the first one after the last)."""
    c = np.sort(np.asarray(clique, dtype=np.int64))
    leaf = np.roll(c, -1)
    inv = 1.0 / scale
    x = src[leaf] - src[c]
    y = (dst[leaf] - dst[c]) * inv
    return Tims(x, y, chain_lanes(c.size))


def complete_tims(src, dst, clique, scale):
    """COMPLETE TIMs of the sorted clique in computeTIMs order (k = i*m - i(i+1)/2 + j-i-1)."""
    c = np.sort(np.asarray(clique, dtype=np.int64))
    m = c.size
    s, d = src[c], dst[c]
    ii, jj = np.triu_indices(m, 1)  # row-major: i ascending, then j ascending == computeTIMs order
    inv = 1.0 / scale
    return Tims(s[jj] - s[ii], (d[jj] - d[ii]) * inv, complete_lanes(m))


def rotation_noise_bound(noise_bound, scale):
    return noise_bound * (2.0 / scale)


# ------------------------------------------------------------------------------------------------ loops
def _div(a, b):
    with np.errstate(all="ignore"):
        return float(np.float64(a) / np.float64(b))


def covariance(t, w):
    """H = sum_k w_k x_k y_k^T in the kernel's per-entry order (a = x*w, then a*y)."""
    a = t.x * w[:, None]
    c = np.empty((t.count, 9))
    for col in range(3):
        for r in range(3):
            c[:, 3 * col + r] = a[:, r] * t.y[:, col]
    h = t.block_sum(c)
    return h.reshape(3, 3).T.copy()  # column-major h[col*3 + r]


def rotation_step(t, w, planar, normalise=True):
    H = covariance(t, w)
    return yaw_rot(H, normalise) if planar else svd_rot(H, normalise)


@np.errstate(over="ignore", invalid="ignore")
def residuals(t, R, planar=False):
    x, y = t.x, t.y
    d0 = y[:, 0] - (R[0, 0] * x[:, 0] + R[0, 1] * x[:, 1] + R[0, 2] * x[:, 2])
    d1 = y[:, 1] - (R[1, 0] * x[:, 0] + R[1, 1] * x[:, 1] + R[1, 2] * x[:, 2])
    if planar:
        return d0 * d0 + d1 * d1
    d2 = y[:, 2] - (R[2, 0] * x[:, 0] + R[2, 1] * x[:, 1] + R[2, 2] * x[:, 2])
    return d0 * d0 + d1 * d1 + d2 * d2


def gnc_tls(t, noise_bound, gnc_factor=1.4, max_iterations=100, cost_threshold=1e-6, planar=False, normalise=True):
    """gnc_tls_block (planar=True: Quatro, yaw only, mask threshold 0.4)."""
    mu = 1.0
    prev_cost = cost = math.inf
    nbsq = noise_bound * noise_bound
    if nbsq < 1e-16:
        nbsq = 1e-2
    w = np.ones(t.count)
    R = np.eye(3)
    it = 0
    for i in range(int(max_iterations)):
        it = i + 1
        R = rotation_step(t, w, planar, normalise)
        r2 = residuals(t, R, planar)
        if i == 0:
            mu = _div(1.0, 2.0 * t.block_max(r2) / nbsq - 1.0)
            if mu <= 0.0:
                break
        th1 = (mu + 1.0) / mu * nbsq
        th2 = mu / (mu + 1.0) * nbsq
        cost = t.block_sum(w * r2)
        with np.errstate(all="ignore"):
            mid = np.sqrt(nbsq * mu * (mu + 1.0) / r2) - mu
        w = np.where(r2 >= th1, 0.0, np.where(r2 <= th2, 1.0, mid))
        cost_diff = abs(cost - prev_cost)
        mu = mu * gnc_factor
        prev_cost = cost
        if cost_diff < cost_threshold:
            break
    mask = w >= (0.4 if planar else 0.5)
    return dict(R=R, cost=cost, iterations=it, weights=w, inliers=mask)


def quatro(t, noise_bound, gnc_factor=1.4, max_iterations=100, cost_threshold=1e-6, normalise=True):
    return gnc_tls(t, noise_bound, gnc_factor, max_iterations, cost_threshold, True, normalise)


def diameter(t, pts, rounded=True):
    """tim_diameter: float(2 sqrt(max |p - mean|^2)) with the mean from block_sum<3> (rounded=False: the double)."""
    c = t.block_sum(pts)
    n = float(t.count)
    g = c / n
    a = pts - g
    d = 2.0 * math.sqrt(t.block_max(a[:, 0] * a[:, 0] + a[:, 1] * a[:, 1] + a[:, 2] * a[:, 2]))
    return float(np.float32(d)) if rounded else d


def fgr(t, noise_bound, gnc_factor=1.4, max_iterations=100, cost_threshold=1e-6, normalise=True):
    """fgr_block: Geman-McClure weights q^2, mask = weight != 0."""
    nbsq = noise_bound * noise_bound
    cost = math.inf
    sd, dd = diameter(t, t.x), diameter(t, t.y)
    gs = sd if sd > dd else dd
    gs = _div(gs, nbsq)
    mu = _div(gs * gs, nbsq)
    w = np.ones(t.count)
    R = np.eye(3)
    it = 0
    with np.errstate(all="ignore"):
        for i in range(int(max_iterations)):
            it = i + 1
            smu = mu * nbsq
            q = smu / (smu + residuals(t, R))
            w = q * q
            R = rotation_step(t, w, False, normalise)
            sq = residuals(t, R)
            cost = t.block_sum((smu * sq) / (smu + sq))
            if cost < cost_threshold or mu < 1.0:
                break
            mu = _div(mu, gnc_factor)
    return dict(R=R, cost=cost, iterations=it, weights=w, inliers=w != 0.0)


def solve(alg, t, noise_bound, gnc_factor=1.4, max_iterations=100, cost_threshold=1e-6, normalise=True):
    """rotation_block: 0 GNC-TLS, 1 FGR, 2 Quatro."""
    if alg == 1:
        return fgr(t, noise_bound, gnc_factor, max_iterations, cost_threshold, normalise)
    return gnc_tls(t, noise_bound, gnc_factor, max_iterations, cost_threshold, alg == 2, normalise)


# ------------------------------------------------------------------------------------------------ exact references
def _mp():
    import mpmath
    mpmath.mp.dps = 60
    return mpmath


def _exact_matrix(H):
    """H as exact mpmath numbers times 2^-e, e the exponent of its largest |entry| (R* does not depend on it)."""
    mp = _mp()
    H = np.asarray(H, dtype=np.float64)
    mx = float(np.abs(H).max())
    e = math.frexp(mx)[1] if mx > 0.0 else 0
    return [[mp.ldexp(mp.mpf(float(H[r, c])), -e) for c in range(3)] for r in range(3)]


def _procrustes_mp(S):
    mp = _mp()
    (xx, xy, xz), (yx, yy, yz), (zx, zy, zz) = S
    N = mp.matrix([[xx + yy + zz, yz - zy, zx - xz, xy - yx],
                   [yz - zy, xx - yy - zz, xy + yx, zx + xz],
                   [zx - xz, xy + yx, -xx + yy - zz, yz + zy],
                   [xy - yx, zx + xz, yz + zy, -xx - yy + zz]])
    E, Q = mp.eigsy(N)
    order = sorted(range(4), key=lambda k: E[k])
    top = order[-1]
    w, x, y, z = (Q[k, top] for k in range(4))
    R = [[w * w + x * x - y * y - z * z, 2 * (x * y - w * z), 2 * (x * z + w * y)],
         [2 * (x * y + w * z), w * w - x * x + y * y - z * z, 2 * (y * z - w * x)],
         [2 * (x * z - w * y), 2 * (y * z + w * x), w * w - x * x - y * y + z * z]]
    return np.array([[float(v) for v in row] for row in R]), E[top], E[top] - E[order[-2]]


def _yaw_mp(S):
    mp = _mp()
    ca, sb = S[0][0] + S[1][1], S[0][1] - S[1][0]
    nrm = mp.sqrt(ca * ca + sb * sb)
    R = np.eye(3)
    if nrm > 0:
        th = mp.atan2(sb, ca)
        c, s = float(mp.cos(th)), float(mp.sin(th))
        R[0, 0], R[0, 1], R[1, 0], R[1, 1] = c, -s, s, c
    return R, nrm, nrm


def procrustes_exact(H):
    """argmax over SO(3) of tr(R H) for H = sum x y^T (Horn's 4x4 matrix N, mpmath.eigsy at 60 digits):
    (R*, lambda_max(N) = max tr(R H), gap lambda_1 - lambda_2; zero gap: the maximiser is not unique)."""
    mp = _mp()
    mx = float(np.abs(np.asarray(H, dtype=np.float64)).max())
    e = math.frexp(mx)[1] if mx > 0.0 else 0
    R, lam, gap = _procrustes_mp(_exact_matrix(H))
    return R, float(mp.ldexp(lam, e)), float(mp.ldexp(gap, e))


def yaw_exact(H):
    """argmax over planar rotations of tr(R2 H2), H2 the top-left 2x2 block (mpmath.atan2): (R*, max, curvature)."""
    mp = _mp()
    mx = float(np.abs(np.asarray(H, dtype=np.float64)).max())
    e = math.frexp(mx)[1] if mx > 0.0 else 0
    R, nrm, _ = _yaw_mp(_exact_matrix(H))
    return R, float(mp.ldexp(nrm, e)), float(mp.ldexp(nrm, e))


def within_exact(R, H, planar=False, k=64.0):
    """Holds R to the exact maximiser: ||R - R*||_F <= k eps ||H||_F / gap where that bound is below 1 (the maximiser
    is unique); otherwise R orthonormal, det R = +1 to 1e-14 and tr(R H) >= max - k eps ||H||_F.  Everything is
    evaluated on H scaled by a power of two in exact arithmetic, so subnormal or huge H are held to the same bound.
    Returns (ok, detail)."""
    mp = _mp()
    S = _exact_matrix(H)
    if planar:
        S = [[S[0][0], S[0][1], mp.mpf(0)], [S[1][0], S[1][1], mp.mpf(0)], [mp.mpf(0)] * 3]
    Rs, lam, gap = (_yaw_mp if planar else _procrustes_mp)(S)
    tol = k * EPS * mp.sqrt(sum(v * v for row in S for v in row))
    if gap > 0 and tol / gap < 1:
        err = float(np.linalg.norm(np.asarray(R, dtype=np.float64) - Rs))
        return err <= tol / gap, f"|R-R*|={err:.3e} bound={float(tol / gap):.3e}"
    R = np.asarray(R, dtype=np.float64)
    orth = float(np.abs(R.T @ R - np.eye(3)).max())
    det = float(np.linalg.det(R))
    val = sum(mp.mpf(float(R[i, j])) * S[j][i] for i in range(3) for j in range(3))
    ok = orth <= 1e-14 and abs(det - 1.0) <= 1e-14 and val >= lam - tol
    return ok, f"orth={orth:.1e} det={det:.17g} tr-max={float(val - lam):.3e} tol={float(tol):.3e} (not unique)"


# ------------------------------------------------------------------------------------------------ test inputs
def random_rotation(rng):
    q = rng.normal(size=4)
    w, x, y, z = q / np.linalg.norm(q)
    return np.array([[w * w + x * x - y * y - z * z, 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), w * w - x * x + y * y - z * z, 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), w * w - x * x - y * y + z * z]])


def axis_rotation(axis, theta):
    a = np.asarray(axis, dtype=np.float64) / np.linalg.norm(axis)
    K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    return np.eye(3) + math.sin(theta) * K + (1 - math.cos(theta)) * (K @ K)


def h_families(seed=0):
    """name -> H (3x3) for the SVD: random, at and near pi, integer ties, permutations, signed diagonals, zero, rank 2
    and 1, reflections with unique / tied / nearly tied smallest singular values, sigma1/sigma3 = 1e16."""
    rng = np.random.default_rng(seed)
    c = {}
    for k in range(4):
        c[f"random{k}"] = rng.normal(size=(3, 3))
    for k in range(2):
        X = rng.normal(size=(3, 40))
        c[f"pi_{k}"] = X @ (axis_rotation(rng.normal(size=3), math.pi) @ X).T
        c[f"pi_minus_1e-7_{k}"] = X @ (axis_rotation(rng.normal(size=3), math.pi - 1e-7) @ X).T
    c["tie_pos"] = np.array([[1.0, 2, 0], [2, 1, 0], [0, 0, 1]])
    c["tie_neg"] = np.array([[1.0, -2, 0], [-2, 1, 0], [0, 0, 1]])
    c["tie_all"] = np.array([[2.0, 1, 1], [1, 2, 1], [1, 1, 2]])
    c["tie_mixed"] = np.array([[3.0, -1, 2], [1, 3, -2], [2, 2, 3]])
    c["skew_int"] = np.array([[3.0, 1, 0], [-1, 3, 0], [0, 0, 1]])
    c["perm_cycle"] = np.array([[0.0, 1, 0], [0, 0, 1], [1, 0, 0]])
    c["perm_swap"] = np.array([[0.0, 1, 0], [1, 0, 0], [0, 0, 1]])
    c["diag_neg"] = np.diag([3.0, -2.0, 1.0])
    c["diag_neg2"] = np.diag([-3.0, -2.0, 1.0])
    c["zero"] = np.zeros((3, 3))
    R = random_rotation(rng)
    for ax in range(3):
        X = rng.normal(size=(3, 30))
        X[ax] = 0.0
        c[f"rank2_{ax}"] = X @ (R @ X).T
    X = np.outer([1.0, 2.0, 3.0], rng.normal(size=30))
    c["rank1"] = X @ (R @ X).T
    Q1, Q2 = random_rotation(rng), random_rotation(rng)
    c["refl_unique"] = Q1 @ np.diag([3.0, 2.0, -1.0]) @ Q2
    c["refl_tied"] = Q1 @ np.diag([2.0, 1.0, -1.0]) @ Q2
    c["refl_tied_exact"] = np.diag([2.0, 1.0, -1.0])
    c["refl_near_tie"] = Q1 @ np.diag([2.0, 1.0, -(1.0 - 1e-9)]) @ Q2
    c["sigma_ratio_1e16"] = Q1 @ np.diag([1e8, 1.0, 1e-8]) @ Q2
    return c


def h2_families():
    """name -> H for the planar closed form (top-left 2x2 block used)."""
    c = {}
    base = np.array([[0.8, 0.6, 0.0], [-0.6, 0.8, 0.0], [0.0, 0.0, 1.0]])
    c["yaw_pi_pos0"] = np.diag([-1.0, -1.0, 1.0])                                     # sb = 0 - 0 = +0.0
    c["yaw_pi_neg0"] = np.array([[-1.0, -0.0, 0.0], [0.0, -1.0, 0.0], [0.0, 0.0, 1.0]])  # sb = -0 - 0 = -0.0
    c["yaw_nrm0"] = np.array([[1.0, 2.0, 5.0], [2.0, -1.0, 0.0], [3.0, 0.0, 1.0]])        # ca = sb = 0
    c["yaw_zero"] = np.zeros((3, 3))
    c["yaw_plain"] = base
    for sc in (1e-160, 1e-170, 1e160, 1e-310, 1e300):
        c[f"yaw_{sc:g}"] = base * sc
    return c


def scale_sweep_h(seed=0):
    """A random H (entries ~1) and, per k, H * 2^k where that is exact; subnormal-range roundings are separate."""
    rng = np.random.default_rng(seed)
    X = rng.normal(size=(3, 20))
    return X @ (random_rotation(rng) @ X).T


def tim_problem(m, outlier_frac, seed, planar=False, noise=1e-3, spread=1.0):
    """m TIMs y = R x + noise, a fraction replaced by random outliers; R a yaw for planar problems."""
    rng = np.random.default_rng(seed)
    R = axis_rotation([0, 0, 1], rng.uniform(-math.pi, math.pi)) if planar else random_rotation(rng)
    x = rng.normal(0, spread, (m, 3))
    y = x @ R.T + rng.normal(0, noise, (m, 3))
    k = int(round(outlier_frac * m))
    idx = rng.permutation(m)[:k]
    y[idx] = rng.normal(0, spread, (k, 3))
    return x, y, R
