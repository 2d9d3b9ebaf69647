"""GPU tests of the batched front end (`pytest -m gpu`): tzr_compute_fpfh_batch and tzr_match_correspondences_batch
must return, per cloud and per pair, bit for bit what the single-cloud / single-pair calls return, with a number of
kernel launches that does not depend on the batch size."""
import importlib
import os
import subprocess

import numpy as np
import pytest

import oracle_lib as orc

capi = importlib.import_module("teaser-plusplus_b200.capi")
synth = importlib.import_module("teaser-plusplus_b200.synth")

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOST = os.path.join(ROOT, "teaser-plusplus_b200", "host")
TOO_LARGE = -6  # TZR_ERR_TOO_LARGE


@pytest.fixture(scope="module")
def ctx():
    c = capi.Context(0)
    yield c
    c.close()


def _same(a, b):
    return np.array_equal(a, b, equal_nan=True)


def _surface(n, seed, shift=(0.5, -0.2, 2.0)):
    rng = np.random.default_rng(seed)
    uv = rng.uniform(-1, 1, size=(n, 2))
    pts = np.stack([uv[:, 0], uv[:, 1], 0.3 * np.sin(3 * uv[:, 0]) * np.cos(2 * uv[:, 1])], axis=1)
    return (pts + rng.normal(scale=0.003, size=pts.shape) + np.array(shift)).astype(np.float32)


def _fpfh_clouds():
    """A ragged batch that takes every path of the radius search."""
    rng = np.random.default_rng(21)
    # points farther apart than the radii: every normal is NaN (fewer than 3 neighbours)
    tiny = [np.arange(3 * k, dtype=np.float32).reshape(k, 3) * np.float32(0.7) for k in (1, 2, 3)]
    dup = rng.uniform(0, 1, size=(600, 3)).astype(np.float32)
    dup[10] = dup[11]                     # duplicate point
    dup[20] = [50, 50, 50]                # isolated
    dup[30] = [np.nan, 0, 0]
    dup[31] = [np.inf, 1, 1]
    brute = _surface(2000, 1)             # below the grid threshold
    g4096 = _surface(4096, 2, shift=(-0.5, 0.2, 2.0))
    g20000 = _surface(20000, 3)
    g20000[17] = [np.nan, 0, 0]
    g20000[18] = [np.inf, 0, 0]
    g20000[19] = [1e6, -1e6, 1e6]
    fallback = _surface(4500, 4)          # a finite point beyond 2^62 cells: the grid cannot index it
    fallback[7] = [1e30, 0, 0]
    bunny, _ = synth.bunny_fpfh()
    return tiny + [dup, brute, g4096, g20000, fallback, bunny.astype(np.float32)]


RN, RF = 0.06, 0.09


@pytest.fixture(scope="module")
def fpfh_singles(ctx):
    clouds = _fpfh_clouds()
    return clouds, [ctx.compute_fpfh(p, RN, RF, return_normals=True) for p in clouds]


@pytest.mark.parametrize("order", ["forward", "reversed"])
def test_fpfh_batch_equals_single_calls(ctx, fpfh_singles, order):
    clouds, singles = fpfh_singles
    idx = list(range(len(clouds)))
    if order == "reversed":
        idx = idx[::-1]
    feats, normals = ctx.compute_fpfh_batch([clouds[i] for i in idx], RN, RF, return_normals=True)
    for k, i in enumerate(idx):
        assert _same(feats[k], singles[i][0]), i
        assert _same(normals[k], singles[i][1]), i
    assert all(np.isnan(normals[idx.index(i)]).all() for i in (0, 1, 2))
    # the descriptors alone (no normals requested) are the same
    assert all(_same(a, b) for a, b in zip(ctx.compute_fpfh_batch([clouds[i] for i in idx], RN, RF), feats))


def test_fpfh_batch_matches_oracle_on_the_bunny(ctx):
    pts, _ = synth.bunny_fpfh()
    feats, normals = ctx.compute_fpfh_batch([_surface(500, 8), pts], 0.03, 0.05, return_normals=True)
    want, wn = orc.compute_fpfh(pts, 0.03, 0.05)
    assert _same(feats[1], want) and _same(normals[1], wn)


def test_fpfh_batch_overflow_marks_only_that_cloud(ctx):
    dense = np.random.default_rng(0).uniform(0, 0.01, size=(5000, 3)).astype(np.float32)
    clouds = [_surface(2000, 5), dense, _surface(500, 6)]
    with pytest.raises(capi.TzrError) as ei:
        ctx.compute_fpfh_batch(clouds, 1.0, 1.0, return_normals=True)
    assert list(ei.value.status) == [0, TOO_LARGE, 0]
    feats, normals = ei.value.result
    for k in (0, 2):
        f, nrm = ctx.compute_fpfh(clouds[k], 1.0, 1.0, return_normals=True)
        assert _same(feats[k], f) and _same(normals[k], nrm)


def _pair(ns, nd, dim, seed, kind="random"):
    """(src_pts, dst_pts, src_feat, dst_feat) of one matcher pair."""
    if dim >= 11:
        mp = synth.matcher_problem(ns, nd, min(ns, nd) // 3, seed=seed, dim=dim)
        sp, tp, sf, tf = mp["src_pts"], mp["dst_pts"], mp["src_feat"], mp["dst_feat"]
    else:
        rng = np.random.default_rng(seed)
        sp, tp = (rng.uniform(0, 1, size=(k, 3)).astype(np.float32) for k in (ns, nd))
        sf, tf = (rng.normal(size=(k, dim)).astype(np.float32) for k in (ns, nd))
    if kind == "ties":      # target descriptors repeated, and every other source equal to one of them
        k = nd // 3
        tf = np.concatenate([tf[:k], tf[:k], tf[:nd - 2 * k]])
        sf = sf.copy()
        m = min(ns, nd)
        sf[:m:2] = tf[:m:2]
    if kind == "nan":       # NaN rows never win
        sf, tf = sf.copy(), tf.copy()
        sf[::7] = np.nan
        tf[3] = np.nan
        tf[5, 0] = np.nan
    return sp, tp, sf, tf


def _matcher_batch(dim):
    pairs = [_pair(900, 700, dim, 1), _pair(700, 900, dim, 2), _pair(64, 64, dim, 3), _pair(1, 1, dim, 4),
             _pair(300, 300, dim, 5, "ties"), _pair(400, 350, dim, 6, "nan"), _pair(3, 2, dim, 7),
             _pair(1500, 1200, dim, 8)]
    seeds = [42, 42, 7, 7, 2**40 + 17, 0, 42, 11]   # equal and distinct seeds
    return pairs, seeds


FLAG_CASES = [(abs_s, cc, tt, ts) for abs_s in (False, True) for cc in (False, True)
              for (tt, ts) in ((False, 0.0), (True, 0.95), (True, 0.0), (False, 0.95))]


@pytest.mark.parametrize("dim", [1, 33, 128])
@pytest.mark.parametrize("abs_scale,crosscheck,tuple_test,tuple_scale", FLAG_CASES)
def test_match_batch_equals_single_calls(ctx, dim, abs_scale, crosscheck, tuple_test, tuple_scale):
    pairs, seeds = _matcher_batch(dim)
    cols = list(zip(*pairs))
    flags = (abs_scale, crosscheck, tuple_test, tuple_scale)
    got, scales = ctx.match_correspondences_batch(*cols, *flags, tuple_seeds=seeds, return_scale=True)
    assert len(got) == len(pairs) == len(scales)
    for b, (p, s) in enumerate(zip(pairs, seeds)):
        want, g = ctx.match_correspondences(*p, *flags, tuple_seed=s, return_scale=True)
        assert np.array_equal(got[b], want), b
        assert np.float32(scales[b]).tobytes() == np.float32(g).tobytes(), b
    if tuple_test and tuple_scale != 0:
        assert len(got[3]) == 0   # ns = nd = 1: the only triple is degenerate, so no correspondence survives


def test_match_batch_equals_oracle(ctx):
    mp = synth.matcher_problem(5000, 4500, 1500, seed=77, feat_noise=0.3)
    a = (mp["src_pts"], mp["dst_pts"], mp["src_feat"], mp["dst_feat"])
    b = _pair(700, 900, 33, 9)
    flags = (False, True, True, 0.95)
    got = ctx.match_correspondences_batch(*zip(b, a), *flags, tuple_seeds=[3, 5])
    assert np.array_equal(got[1], orc.match_correspondences(*a, *flags, tuple_seed=5))
    assert np.array_equal(got[0], orc.match_correspondences(*b, *flags, tuple_seed=3))


def test_match_batch_capacity_too_small(ctx):
    pairs, seeds = _matcher_batch(33)
    cols = list(zip(*pairs))
    singles = [ctx.match_correspondences(*p, False, True, False, 0.0, tuple_seed=s) for p, s in zip(pairs, seeds)]
    cap = [len(p[0]) + len(p[1]) for p in pairs]
    cap[1] = len(singles[1]) - 1
    with pytest.raises(capi.TzrError) as ei:
        ctx.match_correspondences_batch(*cols, False, True, False, 0.0, tuple_seeds=seeds, capacity=cap)
    assert list(ei.value.n_pairs) == [len(s) for s in singles]
    for b, s in enumerate(singles):
        if b == 1:
            assert ei.value.result[b] is None
        else:
            assert np.array_equal(ei.value.result[b], s)


def test_batch_launch_count_does_not_depend_on_b(ctx):
    base = _pair(200, 150, 33, 12)

    def launches(fn):
        l0 = ctx.kernel_launches()
        fn()
        return ctx.kernel_launches() - l0

    for flags in ((False, True, False, 0.0), (False, False, True, 0.95)):
        m2 = launches(lambda: ctx.match_correspondences_batch(*zip(*[base] * 2), *flags, tuple_seeds=[1, 2]))
        m64 = launches(lambda: ctx.match_correspondences_batch(*zip(*[base] * 64), *flags,
                                                               tuple_seeds=list(range(64))))
        assert m2 == m64 > 0
    brute = [_surface(300, 13)]
    grid = [_surface(300, 13), _surface(5000, 14)]
    assert launches(lambda: ctx.compute_fpfh_batch(brute * 2, RN, RF)) == \
        launches(lambda: ctx.compute_fpfh_batch(brute * 64, RN, RF)) > 0
    assert launches(lambda: ctx.compute_fpfh_batch(grid, RN, RF)) == \
        launches(lambda: ctx.compute_fpfh_batch(grid * 32, RN, RF)) > 0


def test_batch_rejects_bad_arguments(ctx):
    p = _pair(10, 10, 33, 1)
    with pytest.raises(capi.TzrError):
        ctx.match_correspondences_batch([p[0]], [p[1]], [p[2]], [p[3][:, :5]])
    big = np.zeros((10, 129), dtype=np.float32)
    with pytest.raises(capi.TzrError):
        ctx.match_correspondences_batch([p[0]], [p[1]], [big], [big])
    with pytest.raises(capi.TzrError):
        ctx.compute_fpfh_batch([_surface(10, 1), np.zeros((0, 3), np.float32)], RN, RF)
    with pytest.raises(capi.TzrError):
        ctx.compute_fpfh_batch([_surface(10, 1)], 0.0, RF)


def test_cpp_facade_batch_equals_consecutive_calls(tmp_path):
    """FPFHEstimation::computeFPFHFeaturesBatch and Matcher::calculateCorrespondencesBatch against consecutive single
    calls (tests/cpp/frontend_batch_test.cc)."""
    subprocess.check_call(["make", "-s", "-C", HOST])
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    exe = str(tmp_path / "frontend_batch_test")
    csrc = os.path.join(ROOT, "teaser-plusplus_b200", "csrc")
    subprocess.check_call([cxx, "-std=c++17", "-O1", "-I", os.path.join(HOST, "include"), "-I",
                           os.path.join(ROOT, "include"), os.path.join(ROOT, "tests", "cpp", "frontend_batch_test.cc"),
                           "-L", HOST, "-lteaser_registration", "-L", csrc, "-lteaser_b200",
                           f"-Wl,-rpath,{HOST}:{csrc}", "-o", exe])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and out.stdout.strip() == "ok", out.stdout + out.stderr
