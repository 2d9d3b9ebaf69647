"""The descriptor front end's arithmetic against exact references, on the CPU through the oracle
(oracle/fpfh_oracle.cc, whose functions the device copies operation for operation; tests/test_gpu_frontend_boundary.py
holds the device to the oracle bit for bit on the same inputs).  References and tolerance rules: frontend_reference.py."""
import math

import numpy as np
import pytest

import frontend_reference as fr
import oracle_lib as orc

# Largest errors of the fixed-sequence elementary functions over the sweeps below, in float32 ulps of the exact value
# (measured: atan2 2.43, acos 1.09, sin 1.36, cos 1.02), pinned with a little room.
ATAN2_MAX_ULP = 2.5
ACOS_MAX_ULP = 1.25
SINCOS_MAX_ULP = 1.5


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def atan2_sweep():
    """Ratios at and around atan's branch points tan(pi/8), tan(3pi/8) and 1 in every quadrant, both as y/1 and 1/x,
    subnormal and huge operands, and random pairs over several magnitudes."""
    ys, xs = [], []
    for t in (math.tan(math.pi / 8), math.tan(3 * math.pi / 8), 1.0):
        for r in fr.float_neighbours(t, 40):
            for sy in (1.0, -1.0):
                for sx in (1.0, -1.0):
                    ys += [sy * r, sy]
                    xs += [sx, sx / r]
    for a, b in [(1e-40, 1.0), (1.0, 1e-40), (-1e-40, -1.0), (1e-40, -1e-40), (1e-45, 3.0), (5.0, 1e-38),
                 (3e38, 1e-3), (1e-3, 3e38), (-2e-39, 7e-39), (1e-30, -1e30)]:
        ys.append(a)
        xs.append(b)
    rng = np.random.default_rng(1)
    g = rng.uniform(-1, 1, (4000, 2)) * 10.0 ** rng.integers(-6, 7, (4000, 2))
    ys += list(g[:, 0])
    xs += list(g[:, 1])
    return np.array(ys, dtype=np.float32), np.array(xs, dtype=np.float32)


def test_atan2_ulp_error():
    y, x = atan2_sweep()
    err = fr.ulp_error(orc.fpfh_elementary("atan2", y, x), fr.exact_atan2(y, x))
    assert err.max() <= ATAN2_MAX_ULP, (err.max(), y[err.argmax()], x[err.argmax()])


def test_atan2_special_values_follow_std_atan2():
    """Signed zeros, both zeros, infinities and NaN give C's atan2 (IEEE 754 / C99 F.9.1.4), rounded to float."""
    vals = [0.0, -0.0, 1.0, -1.0, 2.5e-42, -2.5e-42, np.inf, -np.inf]
    y = np.array([a for a in vals for _ in vals], dtype=np.float32)
    x = np.array([b for _ in vals for b in vals], dtype=np.float32)
    got = orc.fpfh_elementary("atan2", y, x)
    want = np.array([math.atan2(float(a), float(b)) for a, b in zip(y, x)], dtype=np.float32)
    special = (y == 0) | (x == 0) | np.isinf(y) | np.isinf(x)
    assert np.array_equal(_bits(got[special]), _bits(want[special])), \
        [(a, b, g, w) for a, b, g, w in zip(y[special], x[special], got[special], want[special]) if g != w or
         math.copysign(1, g) != math.copysign(1, w)]
    nan = orc.fpfh_elementary("atan2", np.array([np.nan, 1, np.nan], np.float32), np.array([1, np.nan, np.nan],
                                                                                           np.float32))
    assert np.isnan(nan).all()


def test_acos01_ulp_error_and_domain():
    rng = np.random.default_rng(2)
    one = np.float32(1)
    x = np.concatenate([fr.float_neighbours(0.5, 40), rng.uniform(0, 1, 4000),
                        [one - np.float32(k * 2.0 ** -24) for k in range(40)],
                        [0.0, -0.0, 1e-45, 1e-40, 1.2e-38, 1e-20, 1e-4]]).astype(np.float32)
    got = orc.fpfh_elementary("acos01", x)
    err = fr.ulp_error(got, fr.exact_acos(x))
    assert err.max() <= ACOS_MAX_ULP, (err.max(), x[err.argmax()])
    assert got[x == 1][0] == 0.0
    # x > 1 (a dot product of unit vectors that rounded up) and NaN: NaN, like acosf
    bad = np.array([np.nextafter(one, np.float32(2)), 1.5, np.inf, np.nan], dtype=np.float32)
    assert np.isnan(orc.fpfh_elementary("acos01", bad)).all()


def test_sincos_ulp_error_on_the_angle_domain():
    """det_sincos_0_pi2 runs on theta = atan2(...) / 3 in [0, pi/3]: the whole range, the pi/4 switch and the ends."""
    rng = np.random.default_rng(3)
    t = np.concatenate([rng.uniform(0, math.pi / 3, 4000), fr.float_neighbours(math.pi / 4, 20),
                        fr.float_neighbours(math.pi / 3, 5), [0.0, 1e-40, 1e-20, 1e-4]]).astype(np.float32)
    t = t[t >= 0]
    for fn, ref in (("sin", fr.exact_sin), ("cos", fr.exact_cos)):
        err = fr.ulp_error(orc.fpfh_elementary(fn, t), ref(t))
        assert err.max() <= SINCOS_MAX_ULP, (fn, err.max(), t[err.argmax()])


# ---- pair features ------------------------------------------------------------------------------------------------
def axis_pair_cases():
    """Every pair of signed-zero axis normals against displacements along the axes (length 1 and 2, both signs):
    all arithmetic exact, every swap outcome, ties, and f1 at +-pi and +-0."""
    N = fr.signed_axis_normals()
    dps = [s * k * np.eye(3, dtype=np.float32)[ax] for ax in range(3) for s in (1, -1) for k in (1, 2)]
    p1, n1, p2, n2 = [], [], [], []
    base = np.array([3, -1, 2], dtype=np.float32)
    for a in N:
        for b in N:
            for d in dps:
                p1.append(base)
                p2.append(base + d)
                n1.append(a)
                n2.append(b)
    return [np.array(v, dtype=np.float32) for v in (p1, n1, p2, n2)]


def test_pair_features_exact_on_axis_cases():
    p1, n1, p2, n2 = axis_pair_cases()
    f, ok = orc.fpfh_pair_features(p1, n1, p2, n2)
    ref = [fr.pcl_pair_features(*row) for row in zip(p1, n1, p2, n2)]
    want_ok = np.array([r[0] for r in ref])
    want = np.array([[r[1], r[2], r[3]] if r[0] else [0, 0, 0] for r in ref], dtype=np.float32)
    assert np.array_equal(ok, want_ok)
    assert np.array_equal(_bits(f), _bits(want))            # signs of zero included
    bins = np.array([fr.f1_bin(v) for v in f[ok, 0]])
    assert np.array_equal(bins, [fr.f1_bin(r[1]) for r in ref if r[0]])
    # the cases reach f1 = -pi (bin 0), +pi (bin 10) and both zeros (bin 5), and swapped and tied pairs
    f1 = f[ok, 0]
    assert {0, 5, 10} <= set(bins.tolist())
    assert (f1 == -np.float32(math.pi)).any() and (f1 == np.float32(math.pi)).any()
    assert (_bits(f1) == _bits(np.float32(-0.0))).any() and (_bits(f1) == 0).any()
    assert any(r[4] for r in ref) and not all(r[4] for r in ref if r[0])


def test_pair_features_swap_rule_and_values_on_random_pairs():
    """Random points and unit normals: the swap follows acos|angle1| > acos|angle2| evaluated exactly (pairs within
    1e-5 of a tie are left out: their float angles may round either way), and f1, f2, f3 are within a few float ulps of
    the float64 evaluation."""
    rng = np.random.default_rng(4)
    n = 5000
    p1 = rng.normal(size=(n, 3)).astype(np.float32)
    p2 = (p1 + 0.1 * rng.normal(size=(n, 3))).astype(np.float32)
    n1 = rng.normal(size=(n, 3))
    n2 = rng.normal(size=(n, 3))
    n2[: n // 4] = n1[: n // 4] * rng.choice([-1, 1], size=(n // 4, 1))   # parallel normals: |angle1| ~ |angle2|
    n1 = (n1 / np.linalg.norm(n1, axis=1, keepdims=True)).astype(np.float32)
    n2 = (n2 / np.linalg.norm(n2, axis=1, keepdims=True)).astype(np.float32)
    f, ok = orc.fpfh_pair_features(p1, n1, p2, n2)
    assert ok.all()
    ref = np.array([fr.pcl_pair_features(*row)[1:] for row in zip(p1, n1, p2, n2)])
    d = (p2.astype(np.float64) - p1)
    d1 = np.abs((n1 * d).sum(1))
    d2 = np.abs((n2 * d).sum(1))
    clear = np.abs(d1 - d2) > 1e-5 * np.linalg.norm(d, axis=1)
    assert clear.sum() > 0.7 * n
    # the swap is visible in f3's sign convention: f3 = angle1 or -angle2
    swapped = ref[:, 3].astype(bool)
    assert np.array_equal(swapped[clear], (d1 < d2)[clear])
    ang1 = (n1 * d).sum(1) / np.linalg.norm(d, axis=1)
    ang2 = (n2 * d).sum(1) / np.linalg.norm(d, axis=1)
    f3_want = np.where(d1 < d2, -ang2, ang1)
    assert np.abs(f[clear, 2] - f3_want[clear]).max() < 4 * fr.U * 8
    assert np.abs(f[clear, 1] - ref[clear, 1]).max() < 1e-5
    # f1 is an angle near +-pi where a ~ -b: compare on the circle
    df1 = np.abs(np.angle(np.exp(1j * (f[clear, 0] - ref[clear, 0]))))
    assert df1.max() < 1e-4


def test_pair_features_undefined_cases():
    """Coincident points (f4 = 0) and a displacement parallel to the first normal (zero cross product) are not
    defined: ok is False and the row is zero.  A NaN normal gives ok True and NaN f1, f2, f3 (binned to 0 by the SPFH
    kernel)."""
    p = np.zeros((3, 3), dtype=np.float32)
    q = np.array([[0, 0, 0], [0, 0, 2], [1, 0, 0]], dtype=np.float32)
    a = np.array([[0, 0, 1], [0, 0, 1], [np.nan, 0, 0]], dtype=np.float32)
    b = np.array([[1, 0, 0], [0, 0, 1], [0, 1, 0]], dtype=np.float32)
    f, ok = orc.fpfh_pair_features(p, a, q, b)
    assert not ok[0] and not ok[1] and (f[:2] == 0).all()
    # a NaN normal: neither zero test fires (NaN == 0 is false), so the features are "defined" and all three NaN
    assert ok[2] and np.isnan(f[2]).all()


# ---- normals ------------------------------------------------------------------------------------------------------
def _cloud_cases():
    rng = np.random.default_rng(5)
    out = {}
    uv = rng.uniform(-0.5, 0.5, size=(400, 2))
    R = np.linalg.qr(rng.normal(size=(3, 3)))[0]
    out["planar"] = ((np.c_[uv, np.zeros(400)] @ R.T) + [0.2, -0.1, 0.3], 0.2)
    out["curved"] = (np.c_[uv, 0.8 * (uv ** 2).sum(1)] + [0.1, 0.1, -0.4], 0.2)
    out["noisy"] = (np.c_[uv, 0.3 * np.sin(4 * uv[:, 0])] + 0.01 * rng.normal(size=(400, 3)) + [0, 0, 0.5], 0.15)
    return {k: (np.asarray(v, dtype=np.float32), r) for k, (v, r) in out.items()}


@pytest.mark.parametrize("case", ["planar", "curved", "noisy"])
def test_normals_within_the_angle_bound(case):
    pts, r = _cloud_cases()[case]
    _, nrm = orc.compute_fpfh(pts, r, r)
    worst, checked = 0.0, 0
    for q in range(0, len(pts), 3):
        w, V, k, M2 = fr.exact_normal(pts, q, r)
        if k < 3:
            assert np.isnan(nrm[q]).all()
            continue
        cov = np.cov(pts[fr.float_radius_neighbours(pts, q, r)].astype(np.float64).T, bias=True)
        bound = fr.normal_angle_bound(k, M2, np.abs(cov).max(), w[1] - w[0])
        a = fr.angle(nrm[q, :3], V[:, 0])
        assert a <= bound, (q, a, bound)
        assert abs(np.linalg.norm(nrm[q, :3].astype(np.float64)) - 1) < 4 * fr.EPS_F
        # view flip: the normal points to the origin's side of its tangent plane (never strictly away from it)
        assert float(-pts[q].astype(np.float64) @ nrm[q, :3]) >= -bound * np.linalg.norm(pts[q])
        # curvature = lambda_0 / trace, within the eigenvalue error over the trace
        tr = w.sum()
        assert abs(nrm[q, 3] - w[0] / tr) <= 2 * fr.eigenvalue_bound(k, M2, np.abs(cov).max()) / tr + 4 * fr.U
        worst = max(worst, a / bound)
        checked += 1
    assert checked > 100
    print(f"{case}: largest angle / bound = {worst:.3g}")


def test_collinear_and_isotropic_neighbourhoods():
    """A line has no unique normal: only orthogonality to the line is defined (the gap is lambda_2 - lambda_1).  The
    points are dyadic and exactly collinear in float (a line rounded to float is a ribbon whose width is rounding noise,
    and eigen33's cross products of a rank-one matrix's rows are then made of that noise).  Where every cross product
    is exactly zero the normal is 0/0 = NaN, as in PCL.  An isotropic neighbourhood (cube corners) has no normal
    either: unit length and the eigenvalue (curvature 1/3)."""
    d = np.array([0.25, -0.5, 0.5])
    line = (np.outer(np.arange(-10, 11) / 16, d) + [0.25, 0.125, 0.5]).astype(np.float32)
    _, nrm = orc.compute_fpfh(line, 0.3, 0.3)
    finite = 0
    for q in range(len(line)):
        w, V, k, M2 = fr.exact_normal(line, q, 0.3)
        if np.isnan(nrm[q, :3]).any():
            continue
        finite += 1
        b = fr.double_root_angle_bound(w[2], w[2] - w[1]) + fr.normal_angle_bound(k, M2, w[2], w[2] - w[1])
        assert abs(float(nrm[q, :3].astype(np.float64) @ V[:, 2])) <= b
    assert finite >= 3
    # cube corners and centre, rotated so that the float covariance is isotropic only up to rounding (exactly
    # isotropic, every row of A - lambda I is zero and the normal is 0/0 = NaN, as in PCL)
    s = 0.25
    cube = np.array([[x, y, z] for x in (-s, s) for y in (-s, s) for z in (-s, s)] + [[0, 0, 0]])
    R = np.linalg.qr(np.random.default_rng(7).normal(size=(3, 3)))[0]
    cube = (cube @ R.T + 0.5).astype(np.float32)
    _, nrm = orc.compute_fpfh(cube, 1.0, 1.0)
    q = 8
    w, V, k, M2 = fr.exact_normal(cube, q, 1.0)
    assert w[2] - w[0] < 1e-6 * w[0]
    assert abs(np.linalg.norm(nrm[q, :3].astype(np.float64)) - 1) < 4 * fr.EPS_F
    ev_err = fr.triple_root_bound(w[2]) + fr.eigenvalue_bound(k, M2, w[2])
    assert abs(nrm[q, 3] - w[0] / w.sum()) <= 2 * ev_err / w.sum()


def test_exactly_three_neighbours():
    tri = np.array([[0.1, 0.2, 0.3], [0.3, 0.2, 0.35], [0.15, 0.4, 0.2], [5, 5, 5]], dtype=np.float32)
    _, nrm = orc.compute_fpfh(tri, 0.5, 0.5)
    e = np.cross(tri[1] - tri[0], tri[2] - tri[0]).astype(np.float64)
    for q in range(3):
        w, V, k, M2 = fr.exact_normal(tri, q, 0.5)
        assert k == 3
        assert fr.angle(nrm[q, :3], e) <= fr.normal_angle_bound(k, M2, np.abs(w).max(), w[1] - w[0])
    assert np.isnan(nrm[3]).all()


def test_view_flip_at_cos_theta_zero():
    """A 3 x 3 dyadic grid in the plane z = 0 around (1, 0.5, 0): the centre's covariance is exactly diag(a, b, 0),
    eigen33 returns (0, 0, 1), and cos_theta = -p . n is exactly zero, so PCL's `cos_theta < 0` keeps it unflipped.
    The same grid at z = +0.25 has cos_theta < 0 and flips to (0, 0, -1); at z = -0.25 it keeps (0, 0, 1)."""
    g = np.array([[1 + 0.25 * i, 0.5 + 0.25 * j, 0] for i in (-1, 0, 1) for j in (-1, 0, 1)], dtype=np.float32)
    for z, want in ((0.0, 1.0), (0.25, -1.0), (-0.25, 1.0)):
        pts = g + np.array([0, 0, z], dtype=np.float32)
        _, nrm = orc.compute_fpfh(pts, 0.4, 0.4)
        assert np.array_equal(_bits(nrm[4, :2]), _bits([0.0, 0.0])) or z != 0.0
        assert nrm[4, 2] == want, (z, nrm[4])


@pytest.mark.parametrize("k", [20, -20])
def test_power_of_two_scaling_is_exact(k):
    """Scaling a cloud and both radii by 2^k scales every intermediate exactly (no over- or underflow at 2^+-20), and
    eigen33 divides by the largest entry: normals, curvature and descriptors keep their bits."""
    pts, r = _cloud_cases()["noisy"]
    f0, n0 = orc.compute_fpfh(pts, r, 1.5 * r)
    s = np.float32(2.0 ** k)
    f1, n1 = orc.compute_fpfh(pts * s, r * 2.0 ** k, 1.5 * r * 2.0 ** k)
    assert np.array_equal(_bits(n0), _bits(n1)) and np.array_equal(_bits(f0), _bits(f1))


# ---- eigen33 on given matrices -------------------------------------------------------------------------------------
def eigen_cases():
    """Symmetric float32 matrices with a known float64 spectrum: diagonal and axis-permuted (exact), and rotated ones,
    with det(A / max|A|) on both sides of float eps (pcl::computeRoots' switch to computeRoots2), repeated and
    well-separated eigenvalues, at scales 2^+-20."""
    rng = np.random.default_rng(6)
    mats = []
    eps = fr.EPS_F
    for lam in ([2 * eps * 0.8, 0.5, 1.0], [2 * eps * 1.25, 0.5, 1.0], [8 * eps, 0.25, 1.0], [0.0, 0.3, 1.0],
                [1e-3, 0.5, 1.0], [0.1, 0.5, 1.0], [0.2, 0.2, 1.0], [0.05, 0.9, 0.9], [0.3, 0.6, 0.9]):
        for perm in ([0, 1, 2], [2, 0, 1], [1, 2, 0]):
            mats.append(np.diag(np.array(lam)[perm]))
        for _ in range(3):
            Q = np.linalg.qr(rng.normal(size=(3, 3)))[0]
            mats.append(Q @ np.diag(lam) @ Q.T)
    mats = [m * 2.0 ** s for m in mats for s in (0, 20, -20)]
    return np.array(mats, dtype=np.float32)


def check_eigenpairs(cov, ev, vec):
    """ev and vec against the float64 spectrum of the float32 matrices themselves (exact input: no covariance error,
    k = 1 and M2 = 0 in the bound).  In the computeRoots2 branch PCL assumes lambda_0 = 0: the eigenvalue is 0 and the
    vector is that of lambda = 0, off by lambda_0 / gap at most."""
    branches = set()
    for A, e, v in zip(cov.astype(np.float64), ev, vec):
        w, V = np.linalg.eigh(A)
        S = np.abs(A).max()
        br = e == 0.0                      # computeRoots2 sets roots[0] = 0
        if np.count_nonzero(A - np.diag(np.diag(A))) == 0:
            assert br == fr.computeroots2_branch(A), (A, e)   # exact determinant: the switch is where PCL puts it
        branches.add(br)
        dl = w[0] if br else 0.0
        if br:   # taken only when |det(A / S)| < eps (+ its float error), so lambda_0 is that small
            assert w[0] <= 2 * fr.EPS_F * S ** 3 / (w[1] * w[2]) + fr.eigenvalue_bound(0, 0, S), (A, w)
        else:
            repeated = w[1] - w[0] <= 1e-6 * S
            assert abs(e - w[0]) <= fr.eigenvalue_bound(0, 0, S) + (fr.double_root_bound(S) if repeated else 0), \
                (A, e, w)
        assert abs(np.linalg.norm(v.astype(np.float64)) - 1) < 4 * fr.EPS_F
        if w[1] - w[0] > 1e-6 * S:
            assert fr.angle(v, V[:, 0]) <= fr.C_N * (fr.normal_error_scale(0, 0, S) + dl) / (w[1] - w[0]), (A, v, V)
        # lambda_0 repeated: A - lambda I has rank one to within the double root's error, and the cross products of
        # its rows are made of that error (as for the rounded line above): only the eigenvalue and the unit length
        # are defined there
    return branches


def test_smallest_eigenpair_against_eigh():
    cov = eigen_cases()
    ev, vec = orc.fpfh_smallest_eigenpair(cov)
    assert check_eigenpairs(cov, ev, vec) == {True, False}
