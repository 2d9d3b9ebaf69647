"""Exact and float64 references for the descriptor front end (csrc/fpfh.cu, csrc/matcher.cu; DESIGN.md 3.7, 3.8), and
the tolerance rules the tests hold the kernels to.

* Elementary functions: mpmath at 40 digits, errors in float32 ulps of the exact value.
* pcl::computePairFeatures evaluated on inputs whose arithmetic is exact (small integer points, axis-aligned normals
  with signed zeros), in float64 with Python's IEEE atan2, so that signs of zero follow the formulas exactly.
* Normals: the radius neighbour set recomputed in numpy with the kernels' float distance test, then a float64 eigh of
  the two-pass covariance; the angle bound below is what float arithmetic can promise.
* The hashed grid's cell index and hash, replayed in numpy (cell_of, cell_hash)."""
import math

import mpmath
import numpy as np

U = 2.0 ** -24                 # float32 unit roundoff
EPS_F = float(np.finfo(np.float32).eps)

# ---- elementary functions -----------------------------------------------------------------------------------------
mpmath.mp.dps = 40


def ulp32(x):
    """Spacing of float32 at the exact value x (a float or mpf): 2^(e - 23) for |x| in [2^e, 2^(e+1)), subnormal
    spacing below 2^-126."""
    ax = abs(float(x))
    if ax < 2.0 ** -126:
        return 2.0 ** -149
    return 2.0 ** (math.frexp(ax)[1] - 1 - 23)


def ulp_error(got, exact):
    """|got - exact| in float32 ulps of exact, per element (exact as mpf values)."""
    return np.array([float(abs(mpmath.mpf(float(g)) - e)) / ulp32(e) for g, e in zip(got, exact)])


def exact_atan2(y, x):
    return [mpmath.atan2(mpmath.mpf(float(a)), mpmath.mpf(float(b))) for a, b in zip(y, x)]


def exact_acos(x):
    return [mpmath.acos(mpmath.mpf(float(a))) for a in x]


def exact_sin(x):
    return [mpmath.sin(mpmath.mpf(float(a))) for a in x]


def exact_cos(x):
    return [mpmath.cos(mpmath.mpf(float(a))) for a in x]


def float_neighbours(v, k):
    """v and its k float32 neighbours on each side."""
    v = np.float32(v)
    out = [v]
    up, dn = v, v
    for _ in range(k):
        up = np.nextafter(up, np.float32(np.inf))
        dn = np.nextafter(dn, np.float32(-np.inf))
        out += [up, dn]
    return np.array(out, dtype=np.float32)


# ---- pcl::computePairFeatures, exactly ------------------------------------------------------------------------------
def bin11(v):
    """The histogram bin of the SPFH kernel and the oracle: floor(v) clamped to [0, 10], NaN -> 0."""
    if v != v:
        return 0
    f = math.floor(v)
    return 0 if f < 0 else 10 if f >= 11 else int(f)


D_PI = float(np.float32(1.0) / (np.float32(2.0) * np.float32(math.pi)))   # the kernels' float 1 / (2 pi)


def f1_bin(f1):
    return bin11(11 * ((float(f1) + math.pi) * D_PI))


def pcl_pair_features(p1, n1, p2, n2):
    """computePairFeatures (features/src/pfh_tools.cpp) in float64 with the operation order of the source and IEEE
    signed zeros (math.atan2 is C's atan2).  When every input is a small integer and the normals are axis-aligned, each
    product and sum is exact in float32 as well, so this is the exact value the float code must give, sign of zero
    included.  Returns (ok, f1, f2, f3, swapped); the swap is decided exactly as acos|angle1| > acos|angle2|, i.e.
    |n1 . dp| < |n2 . dp| (acos is strictly decreasing and both angles share f4)."""
    p1, n1, p2, n2 = ([float(c) for c in v] for v in (p1, n1, p2, n2))
    dp = [p2[k] - p1[k] for k in range(3)]
    f4 = math.sqrt(dp[0] * dp[0] + dp[1] * dp[1] + dp[2] * dp[2])
    if f4 == 0.0:
        return False, 0.0, 0.0, 0.0, False
    a, b = list(n1), list(n2)
    d1 = a[0] * dp[0] + a[1] * dp[1] + a[2] * dp[2]
    d2 = b[0] * dp[0] + b[1] * dp[1] + b[2] * dp[2]
    swapped = abs(d1) < abs(d2)
    if swapped:
        a, b = list(n2), list(n1)
        dp = [-c for c in dp]
        f3 = -(d2 / f4)
    else:
        f3 = d1 / f4
    v = [dp[1] * a[2] - dp[2] * a[1], dp[2] * a[0] - dp[0] * a[2], dp[0] * a[1] - dp[1] * a[0]]
    vn = math.sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2])
    if vn == 0.0:
        return False, 0.0, 0.0, 0.0, swapped
    v = [c / vn for c in v]
    w = [a[1] * v[2] - a[2] * v[1], a[2] * v[0] - a[0] * v[2], a[0] * v[1] - a[1] * v[0]]
    f2 = v[0] * b[0] + v[1] * b[1] + v[2] * b[2]
    f1 = math.atan2(w[0] * b[0] + w[1] * b[1] + w[2] * b[2], a[0] * b[0] + a[1] * b[1] + a[2] * b[2])
    return True, f1, f2, f3, swapped


def signed_axis_normals():
    """Every unit axis vector with every sign pattern of its two zero components: 24 normals."""
    out = []
    for ax in range(3):
        for s in (1.0, -1.0):
            for z1 in (0.0, -0.0):
                for z2 in (0.0, -0.0):
                    v = [z1, z2]
                    v.insert(ax, s)
                    out.append(v)
    return np.array(out, dtype=np.float32)


# ---- normals ------------------------------------------------------------------------------------------------------
def float_radius_neighbours(pts, q, r):
    """Indices of the points the kernels' float test accepts for query q: d = dx*dx; d += dy*dy; d += dz*dz in
    float32, d < (float)(r*r)."""
    p = np.asarray(pts, dtype=np.float32)
    d = (p - p[q]).astype(np.float32)
    s = (d[:, 0] * d[:, 0]).astype(np.float32)
    s = (s + (d[:, 1] * d[:, 1]).astype(np.float32)).astype(np.float32)
    s = (s + (d[:, 2] * d[:, 2]).astype(np.float32)).astype(np.float32)
    with np.errstate(invalid="ignore"):
        return np.nonzero(s < np.float32(r * r))[0]


def exact_normal(pts, q, r):
    """Float64 reference of point q's normal: (eigenvalues ascending, eigenvectors, neighbour count, M2) of the biased
    covariance of its float-test neighbours, M2 = max ||p||^2 over them."""
    nb = float_radius_neighbours(pts, q, r)
    P = np.asarray(pts, dtype=np.float64)[nb]
    c = P - P.mean(0)
    w, V = np.linalg.eigh(c.T @ c / len(nb))
    return w, V, len(nb), float((P ** 2).sum(1).max())


# Angle bound.  The kernels form the covariance in one float pass, E[p p^T] - E[p] E[p]^T over raw coordinates
# (PCL <= 1.11).  Each of the k-term sequential sums has error <= (k - 1) u sum|t| (Higham 3.1); with the products
# and the division by k, E[x y] is within (k + 1) u M2, each mean within k u sqrt(M2) and so E[x] E[y] within
# (2k + 1) u M2, and the subtraction adds 2 u M2: (3k + 4) u M2 per entry, M2 = max ||p||^2, and
# ||E1||_2 <= ||E1||_F <= 3 (3k + 4) u M2.  pcl::eigen33 then returns the
# smallest root to within c u S of the perturbed matrix (S = max |entry|: the trigonometric roots of the scaled matrix
# carry a few roundings of numbers of size one) and the normal as the largest cross product of two rows of
# A - lambda I, whose direction moves by at most c' (delta lambda + u S) / gap.  With the Davis-Kahan sin(theta)
# theorem for E1, the angle between the computed and the exact normal obeys
#     sin(angle) <= C_N u (3 (3k + 4) M2 + S) / gap,   gap = lambda_1 - lambda_0.
# C_N = 8 covers the constants with room; the CPU test shows the oracle meets it on every case (the largest ratio of
# measured angle to bound is printed there), so C_N is set by the arithmetic and not by the device.
C_N = 8.0


def normal_error_scale(k, M2, S):
    """u (3 (3k + 4) M2 + S): the float error of the covariance and of the eigen solver, in covariance units."""
    return U * (3 * (3 * k + 4) * M2 + S)


def normal_angle_bound(k, M2, S, gap):
    return C_N * normal_error_scale(k, M2, S) / gap


def eigenvalue_bound(k, M2, S):
    """|ev - lambda_0| (Weyl for the covariance error, plus the solver's root error)."""
    return C_N * normal_error_scale(k, M2, S)


# Multiple roots.  pcl::eigen33 finds lambda_0 as a root of the characteristic cubic, and a root of multiplicity m
# moves by (u S)^(1/m) S^(1 - 1/m) when the coefficients move by u S (a polynomial's multiple roots are
# ill-conditioned).  A repeated smallest eigenvalue (a line, whose two smallest are both 0) therefore comes out only
# to sqrt(u) S, and A - lambda I then has rows off by that much, so the normal is orthogonal to the remaining
# eigenvector only within C_N sqrt(u) S / (lambda_2 - lambda_1); a triple root (an isotropic neighbourhood) is
# found to u^(1/3) S.
def double_root_bound(S):
    return C_N * math.sqrt(U) * S


def double_root_angle_bound(S, gap):
    return double_root_bound(S) / gap


def triple_root_bound(S):
    return C_N * U ** (1.0 / 3.0) * S


def angle(u, v):
    """Unsigned angle between the lines of u and v (normals are defined up to sign before the view flip)."""
    u = np.asarray(u, dtype=np.float64)
    v = np.asarray(v, dtype=np.float64)
    c = abs(float(u @ v)) / (np.linalg.norm(u) * np.linalg.norm(v))
    return math.acos(min(1.0, c))


def computeroots2_branch(cov):
    """Whether pcl::computeRoots takes the computeRoots2 branch: |det(cov / max|cov|)| < float eps (float64 value of
    the determinant; the tests keep it well away from the threshold on each side)."""
    m = np.asarray(cov, dtype=np.float64)
    return abs(np.linalg.det(m / np.abs(m).max())) < EPS_F


# ---- hashed grid (fpfh.cu cell_of / cell_hash) ----------------------------------------------------------------------
def cell_edge(normal_radius, fpfh_radius):
    return max(normal_radius, fpfh_radius) * (1.0 + 1e-5)


def cell_index(x, origin, h):
    """floor(((double)x - o) * (1 / h)) per coordinate, the device's double arithmetic."""
    return np.floor((np.asarray(x, dtype=np.float32).astype(np.float64) - np.float64(origin)) * (1.0 / h))


def cell_hash(ix, iy, iz, mask):
    m32 = 0xffffffff
    h = ((int(ix) * 73856093) & m32) ^ ((int(iy) * 19349663) & m32) ^ ((int(iz) * 83492791) & m32)
    return h & mask


NEIGHBOUR_OFFSETS = [(t % 3 - 1, (t // 3) % 3 - 1, t // 9 - 1) for t in range(27)]


def repeated_bucket_cell(mask, lo=1, hi=64):
    """A cell (ix, iy, iz) whose own bucket is also the bucket of another of its 26 neighbours, so that a query there
    reaches its own points twice unless the 27 buckets are de-duplicated."""
    for ix in range(lo, hi):
        for iy in range(lo, hi):
            for iz in range(lo, hi):
                own = cell_hash(ix, iy, iz, mask)
                for d in NEIGHBOUR_OFFSETS:
                    if d != (0, 0, 0) and cell_hash(ix + d[0], iy + d[1], iz + d[2], mask) == own:
                        return (ix, iy, iz), d
    raise AssertionError("no repeated bucket in the searched range")


# ---- matcher ------------------------------------------------------------------------------------------------------
def l2_error_bound(q, db):
    """Bound on |fl32(L2(q, x)) - L2(q, x)| for every row x of db, flann::L2<float>'s order: each squared difference
    carries 2 roundings, and the grouped sum of dim terms at most dim - 1 more, so (dim + 2) u sum (q - x)^2 with the
    float64 sum standing in for the exact one (its own error is negligible at u^2)."""
    q = np.asarray(q, dtype=np.float64)
    d64 = ((np.asarray(db, dtype=np.float64) - q) ** 2).sum(1)
    return (q.size + 2) * U * d64, d64
