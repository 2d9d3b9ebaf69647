"""The descriptor front end at its edges on the device (`pytest -m gpu`): the building blocks bit for bit against the
oracle on any input, and the hashed-grid radius search bit for bit against brute force where a grid can go wrong
(cell boundaries, far points, repeated buckets, the size switch, the neighbour cap), with the route chosen per call by
the debug flags 4194304 (brute force) and 8388608 (grid).  References: frontend_reference.py."""
import importlib

import numpy as np
import pytest

import frontend_reference as fr
import oracle_lib as orc
from test_frontend_reference_cpu import axis_pair_cases, check_eigenpairs, eigen_cases

capi = importlib.import_module("teaser-plusplus_b200.capi")

pytestmark = pytest.mark.gpu

BRUTE, GRID = capi.FLAG_FPFH_BRUTE_FORCE, capi.FLAG_FPFH_GRID


@pytest.fixture(scope="module")
def ctx():
    c = capi.Context(0)
    yield c
    c.close()


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def _same(a, b):
    """Bit for bit (signs of zero included), except that any NaN equals any NaN: the device's NaN constant and the
    host's quiet NaN differ in their payload bits."""
    a, b = np.asarray(a, dtype=np.float32), np.asarray(b, dtype=np.float32)
    na, nb = np.isnan(a), np.isnan(b)
    return a.shape == b.shape and np.array_equal(na, nb) and np.array_equal(_bits(a[~na]), _bits(b[~nb]))


def all_routes(ctx, pts, rn, rf):
    """Descriptors and normals by size (default), brute force and the grid, each bit-equal to the oracle."""
    want_f, want_n = orc.compute_fpfh(pts, rn, rf)
    try:
        for flags in (0, BRUTE, GRID):
            ctx.set_flags(flags)
            f, n = ctx.compute_fpfh(pts, rn, rf, return_normals=True)
            assert _same(n, want_n), (flags, np.argwhere(~(_bits(n) == _bits(want_n)).all(1))[:5].ravel())
            assert _same(f, want_f), (flags, np.argwhere(~(_bits(f) == _bits(want_f)).all(1))[:5].ravel())
    finally:
        ctx.set_flags(0)
    return want_f, want_n


# ---- building blocks ------------------------------------------------------------------------------------------------
def pair_feature_inputs():
    p1, n1, p2, n2 = axis_pair_cases()
    rng = np.random.default_rng(11)
    m = 4000
    q1 = rng.normal(size=(m, 3)).astype(np.float32)
    q2 = (q1 + 0.05 * rng.normal(size=(m, 3))).astype(np.float32)
    a = rng.normal(size=(m, 3))
    b = rng.normal(size=(m, 3))
    b[:1000] = a[:1000] * rng.choice([-1, 1], size=(1000, 1))
    a = (a / np.linalg.norm(a, axis=1, keepdims=True)).astype(np.float32)
    b = (b / np.linalg.norm(b, axis=1, keepdims=True)).astype(np.float32)
    # angles around acos's switch at 0.5 and near 1, coincident points, NaN normals, subnormal displacements
    d = np.array([0, 0, 1], dtype=np.float32)
    for c in list(fr.float_neighbours(0.5, 8)) + list(fr.float_neighbours(1.0, 4)):
        s = np.sqrt(max(0.0, 1 - float(c) ** 2))
        q1 = np.vstack([q1, [[0, 0, 0]]]).astype(np.float32)
        q2 = np.vstack([q2, [d]]).astype(np.float32)
        a = np.vstack([a, [[s, 0, c]]]).astype(np.float32)
        b = np.vstack([b, [[0, s, -c]]]).astype(np.float32)
    extra = [([0, 0, 0], [0, 0, 1], [0, 0, 0], [1, 0, 0]), ([0, 0, 0], [np.nan, 0, 0], [1, 0, 0], [0, 1, 0]),
             ([0, 0, 0], [0, 0, 1], [1e-42, 0, 0], [0, 1, 0]), ([1, 2, 3], [0, 0, 1], [1, 2, 5], [0, 0, 1])]
    for e in extra:
        q1, a, q2, b = (np.vstack([x, [v]]).astype(np.float32) for x, v in zip((q1, a, q2, b), e))
    return [np.vstack([u, v]).astype(np.float32) for u, v in zip((p1, n1, p2, n2), (q1, a, q2, b))]


def test_pair_features_bit_exact(ctx):
    ins = pair_feature_inputs()
    f, ok = ctx.fpfh_pair_features(*ins)
    wf, wok = orc.fpfh_pair_features(*ins)
    assert np.array_equal(ok, wok)
    assert _same(f, wf)
    # a dense random sweep: a one-ulp change of one polynomial coefficient moves about 3e-5 of the results
    rng = np.random.default_rng(21)
    m = 1_000_000
    dense = [rng.normal(size=(m, 3)).astype(np.float32) for _ in range(4)]
    df, dok = ctx.fpfh_pair_features(*dense)
    wdf, wdok = orc.fpfh_pair_features(*dense)
    assert np.array_equal(dok, wdok) and _same(df, wdf)
    # and equal to PCL's formulas, exactly, on the axis cases (signs of zero and the f1 bins at +-pi included)
    n_axis = len(axis_pair_cases()[0])
    for i in range(0, n_axis, 7):
        r = fr.pcl_pair_features(*(x[i] for x in ins))
        assert ok[i] == r[0]
        if r[0]:
            assert _same(f[i], np.array(r[1:4], dtype=np.float32))


def test_smallest_eigenpair_bit_exact(ctx):
    cov = eigen_cases()
    rng = np.random.default_rng(12)
    X = rng.normal(size=(3000, 3, 3)) * 10.0 ** rng.integers(-8, 8, (3000, 1, 1))
    rand = (X + X.transpose(0, 2, 1)).astype(np.float32)
    allc = np.concatenate([cov, rand, np.zeros((1, 3, 3), np.float32), np.eye(3, dtype=np.float32)[None]])
    ev, vec = ctx.fpfh_smallest_eigenpair(allc)
    wev, wvec = orc.fpfh_smallest_eigenpair(allc)
    assert _same(ev, wev) and _same(vec, wvec)
    assert check_eigenpairs(cov, ev[:len(cov)], vec[:len(cov)]) == {True, False}


@pytest.mark.parametrize("k", [20, -20])
def test_power_of_two_scaling_keeps_bits(ctx, k):
    rng = np.random.default_rng(13)
    uv = rng.uniform(-0.5, 0.5, size=(1500, 2))
    pts = (np.c_[uv, 0.3 * np.sin(4 * uv[:, 0])] + 0.01 * rng.normal(size=(1500, 3)) + [0, 0, 0.5]).astype(np.float32)
    f0, n0 = ctx.compute_fpfh(pts, 0.1, 0.15, return_normals=True)
    f1, n1 = ctx.compute_fpfh(pts * np.float32(2.0 ** k), 0.1 * 2.0 ** k, 0.15 * 2.0 ** k, return_normals=True)
    assert _same(n0, n1) and _same(f0, f1)


# ---- radius search: grid against brute force ---------------------------------------------------------------------
def triples(centres, r, axis=0, sep=0.99999):
    """At every centre c: c, c + sep r along the axis and a third point 0.58 r from both (so normals are defined)."""
    e = np.eye(3)[axis]
    o = np.eye(3)[(axis + 1) % 3]
    c = np.asarray(centres, dtype=np.float64)
    a = c.astype(np.float32)
    b = (a.astype(np.float64) + sep * r * e).astype(np.float32)
    t = (a.astype(np.float64) + 0.5 * r * e + 0.3 * r * o).astype(np.float32)
    return np.concatenate([a, b, t])


def test_cell_boundaries(ctx):
    """Points on and around the planes x, y, z = origin + k h (both float neighbours of each plane), and pairs
    r (1 - 2^-20) apart that straddle one, in a cloud of a few thousand points searched by grid and brute force."""
    rn, rf = 0.05, 0.08
    h = fr.cell_edge(rn, rf)
    rng = np.random.default_rng(14)
    pts = [np.zeros((1, 3))]                                    # the origin: the grid's cell k starts at k h
    for axis in range(3):
        for k in range(1, 40, 3):
            plane = k * h
            base = rng.uniform(0.1, 3.0, size=(3,))
            for v in fr.float_neighbours(plane, 2):
                p = base.copy()
                p[axis] = v
                pts.append(p[None])
            c = base.copy()
            c[axis] = plane - 0.4 * rf
            pts.append(triples([c], rf, axis, 1 - 2.0 ** -20).astype(np.float64))
    pts.append(rng.uniform(0, 3, size=(2000, 3)))
    pts = np.concatenate(pts).astype(np.float32)
    all_routes(ctx, pts, rn, rf)


FAR = [(-1e8, 0.01), (-3e7, 0.01), (-1e11, 0.01), (-1e12, 0.05), (-1e17, 0.1), (-3.2e38, 0.05), (3.2e38, 0.05)]


@pytest.mark.parametrize("far,r", FAR)
def test_far_point(ctx, far, r):
    """Triples 0.99999 r apart near the origin and three mutual neighbours near x = far.  With the origin at far < 0
    the double cell index is off by more than the margin from about 2^33 cells on (1e11 / 0.01 and beyond), and such a
    cloud must fall back to brute force; 3e7 / 0.01 (under 2^32 cells) stays on the grid.  The replay below shows which
    of these clouds hold true neighbours that the grid, indexing them, would put two cells apart.  At +-3.2e38 the far
    points must be in the bounding box and the fallback too: they find each other (their normals are NaN, x^2
    overflows, but their descriptors count the pairs), where a grid that left them out would give them empty ones."""
    o, h = np.float32(min(far, 0.0)), fr.cell_edge(r, r)
    cand = np.arange(200000) * (r / 997.0)
    a = cand.astype(np.float32)
    b = (a.astype(np.float64) + 0.99999 * r).astype(np.float32)
    apart = np.abs(fr.cell_index(b, o, h) - fr.cell_index(a, o, h))
    if far in (-1e11, -1e12, -1e17):
        assert (apart > 1).sum() > 0      # the case reaches the gap the guard closes
    elif far in (-1e8, -3e7):
        assert (apart <= 1).all()
    xs = np.concatenate([cand[apart > 1][:300], cand[:1500]])[:1500]
    m = len(xs)
    centres = np.c_[xs, (np.arange(m) % 50) * 3 * r, (np.arange(m) // 50) * 3 * r]
    cluster = [[far, 0, 0], [far, 0.4 * r, 0], [far, 0, 0.4 * r]]
    pts = np.concatenate([triples(centres, r), cluster]).astype(np.float32)
    f, n = all_routes(ctx, pts, r, r)
    assert np.isfinite(n[:3 * m]).all()
    assert (f[-3:].sum(1) > 0).all()


def test_cell_margin_is_needed(ctx):
    """Each point paired with the farthest float along x that still passes the float test d^2 < r^2, with the origin at
    -4.2e7 (r = 0.01: 4.2e9 cells, under the 2^32 limit, so the grid is used).  The replay selects pairs that a cell
    edge of exactly r would put two cells apart; the 1e-5 margin of the edge keeps them in adjacent cells."""
    r = 0.01
    o = np.float32(-4.2e7)
    cand = np.arange(200000) * (r / 997.0)
    a = cand.astype(np.float32)
    b = (a.astype(np.float64) + r).astype(np.float32)
    r2 = np.float32(r * r)
    for _ in range(8):
        d = (b - a).astype(np.float32)
        b = np.where((d * d).astype(np.float32) < r2, b, np.nextafter(b, np.float32(-np.inf)))
    d = (b - a).astype(np.float32)
    assert ((d * d).astype(np.float32) < r2).all()
    need = np.abs(fr.cell_index(b, o, r) - fr.cell_index(a, o, r)) > 1
    assert need.sum() >= 1
    assert (np.abs(fr.cell_index(b, o, fr.cell_edge(r, r)) - fr.cell_index(a, o, fr.cell_edge(r, r))) <= 1).all()
    xs = np.concatenate([a[need], a[:1000]])
    pb = np.concatenate([b[need], b[:1000]])
    m = len(xs)
    y, z = (np.arange(m) % 40) * 3 * r, (np.arange(m) // 40) * 3 * r
    pts = np.concatenate([np.c_[xs, y, z], np.c_[pb, y, z], np.c_[xs + 0.5 * r, y + 0.3 * r, z], [[o, 0, 0]]])
    all_routes(ctx, pts.astype(np.float32), r, r)


def test_far_point_default_route(ctx):
    """The same at grid size without the flag: 6000 points plus one at -1e12 (r = 0.05)."""
    r = 0.05
    xs = np.arange(2000) * (r / 997.0)
    centres = np.c_[xs, (np.arange(2000) % 50) * 3 * r, (np.arange(2000) // 50) * 3 * r]
    pts = np.concatenate([triples(centres, r), [[-1e12, 0, 0]]]).astype(np.float32)
    assert len(pts) >= 4096
    all_routes(ctx, pts, r, r)


def test_repeated_buckets_are_visited_once(ctx):
    """A small cloud on the grid (flag 8388608: 1024 buckets) whose points sit in a cell that shares its bucket with
    one of its 26 neighbour cells: without the de-duplication of the 27 buckets, each point would be its own and its
    neighbours' neighbour twice."""
    r = 0.1
    h = fr.cell_edge(r, r)
    (ix, iy, iz), d = fr.repeated_bucket_cell(1023)
    centre = (np.array([ix, iy, iz]) + 0.5) * h
    rng = np.random.default_rng(15)
    cluster = centre + rng.uniform(-0.3 * h, 0.3 * h, size=(12, 3))
    other = (np.array([ix, iy, iz]) + np.array(d) + 0.5) * h + rng.uniform(-0.3 * h, 0.3 * h, size=(6, 3))
    pts = np.concatenate([[[0, 0, 0]], cluster, other, rng.uniform(0, 30 * h, size=(300, 3))]).astype(np.float32)
    assert fr.cell_index(pts[1:13], 0.0, h).tolist() == [[ix, iy, iz]] * 12
    all_routes(ctx, pts, r, r)


@pytest.mark.parametrize("n", [4095, 4096, 4097])
def test_route_switch_sizes(ctx, n):
    rng = np.random.default_rng(n)
    uv = rng.uniform(-1, 1, size=(n, 2))
    pts = (np.c_[uv, 0.3 * np.sin(3 * uv[:, 0]) * np.cos(2 * uv[:, 1])] + rng.normal(scale=0.003, size=(n, 3))
           + [0.5, -0.2, 2.0]).astype(np.float32)
    all_routes(ctx, pts, 0.06, 0.09)


@pytest.mark.parametrize("flags", [0, BRUTE, GRID])
def test_ragged_batch_mixing_routes(ctx, flags):
    """Grid clouds, brute-force clouds and a grid-size cloud that falls back (a far point) in one batch: every cloud
    equals its single call and the oracle."""
    rng = np.random.default_rng(16)

    def surf(n, off):
        uv = rng.uniform(-1, 1, size=(n, 2))
        return (np.c_[uv, 0.2 * np.sin(3 * uv[:, 0])] + rng.normal(scale=0.003, size=(n, 3)) + off).astype(np.float32)

    fallback = surf(4500, [0, 0, 1])
    fallback[77] = [-1e12, 0, 0]
    clouds = [surf(5000, [0.5, 0, 2]), surf(700, [0, 0, 1]), fallback, surf(3, [0, 0, 1]), surf(4096, [1, 1, 1]),
              surf(1, [0, 0, 0])]
    rn, rf = 0.07, 0.1
    try:
        ctx.set_flags(flags)
        got, nrm = ctx.compute_fpfh_batch(clouds, rn, rf, return_normals=True)
    finally:
        ctx.set_flags(0)
    for c, g, nr in zip(clouds, got, nrm):
        wf, wn = orc.compute_fpfh(c, rn, rf)
        assert _same(g, wf) and _same(nr, wn)


@pytest.mark.parametrize("flags", [0, BRUTE, GRID])
def test_neighbour_cap(ctx, flags):
    """4096 points within one radius of each other: exactly 4096 neighbours each is accepted; one more point is
    TZR_ERR_TOO_LARGE for that cloud only."""
    rng = np.random.default_rng(17)
    ball = rng.uniform(-0.01, 0.01, size=(4097, 3)).astype(np.float32) + np.float32(0.5)
    small = rng.uniform(0, 1, size=(300, 3)).astype(np.float32)
    try:
        ctx.set_flags(flags)
        f, n = ctx.compute_fpfh(ball[:4096], 0.5, 0.5, return_normals=True)
        with pytest.raises(capi.TzrError) as e:
            ctx.compute_fpfh_batch([ball, small], 0.5, 0.5)
    finally:
        ctx.set_flags(0)
    wf, wn = orc.compute_fpfh(ball[:4096], 0.5, 0.5)
    assert _same(f, wf) and _same(n, wn)
    assert e.value.status.tolist() == [-6, 0]
    assert _same(e.value.result[1], orc.compute_fpfh(small, 0.5, 0.5)[0])


# ---- matcher ------------------------------------------------------------------------------------------------------
def test_feature_nn_winner_within_the_l2_bound(ctx):
    """The float32 winner is a float64 nearest neighbour to within the float error of the two distances."""
    rng = np.random.default_rng(18)
    q = rng.uniform(0, 1, size=(500, 33)).astype(np.float32)
    db = rng.uniform(0, 1, size=(3000, 33)).astype(np.float32)
    db[1000:1500] = db[:500] + rng.normal(scale=1e-4, size=(500, 33)).astype(np.float32)   # near ties
    idx, dist = ctx.feature_nn(q, db)
    for i in range(len(q)):
        bound, d64 = fr.l2_error_bound(q[i], db)
        j = d64.argmin()
        assert d64[idx[i]] <= d64[j] + bound[idx[i]] + bound[j]
        assert abs(float(dist[i]) - d64[idx[i]]) <= bound[idx[i]]


def test_feature_nn_nonfinite_queries(ctx):
    rng = np.random.default_rng(19)
    q = rng.uniform(0, 1, size=(8, 33)).astype(np.float32)
    db = rng.uniform(0, 1, size=(200, 33)).astype(np.float32)
    q[0, :] = np.nan
    q[1, 5] = np.nan
    q[2, :] = np.inf
    q[3, 7] = -np.inf
    db[50, 7] = -np.inf
    db[60, :] = np.inf
    idx, _ = ctx.feature_nn(q, db)
    assert np.array_equal(idx, orc.nn1(q, db))


@pytest.mark.parametrize("ndb", [63, 64, 65, 127, 128, 129, 40000, 70001])
def test_feature_nn_tile_edges_and_segment_splits(ctx, ndb):
    """Database sizes at the 64-row tile edges and past the host's segment splits.  tzr_feature_nn cuts the database
    into segments of whole 64-row tiles (nn_work_append), so every split is a tile edge whatever the device's SM count:
    a query's exact copy is placed on both sides of every tile edge (edge e serves query e mod nq), and the lowest index
    among a query's copies must win, across tiles and across segments merged by the atomic minimum."""
    rng = np.random.default_rng(ndb)
    nq = 70
    q = rng.uniform(0, 1, size=(nq, 33)).astype(np.float32)
    db = rng.uniform(0, 1, size=(ndb, 33)).astype(np.float32)
    first = {}
    for e, s in enumerate(range(64, ndb, 64)):
        i = e % nq
        db[s - 1] = q[i]
        db[s] = q[i]
        first.setdefault(i, s - 1)
    idx, _ = ctx.feature_nn(q, db)
    assert np.array_equal(idx, orc.nn1(q, db))
    for i, lo in first.items():
        assert idx[i] == lo
