"""CPU checks of tests/matcher_reference.py: it equals the oracle's restatement, its sequential sum and draws are
what they claim, and every premise tests/test_gpu_matcher_boundary.py builds on holds."""
import importlib
import itertools

import numpy as np
import pytest

import matcher_reference as mr
import oracle_lib as orc

synth = importlib.import_module("teaser-plusplus_b200.synth")
F32 = np.float32

FLAG_CASES = [(abs_s, cc, tt, ts) for abs_s in (False, True) for cc in (False, True)
              for (tt, ts) in ((False, 0.0), (True, 0.95), (True, 0.0), (False, 0.95))]


@pytest.mark.parametrize("ns,nd,nc", [(90, 70, 30), (70, 90, 30), (64, 64, 64), (100, 100, 0), (3, 2, 2),
                                      (1, 1, 1), (300, 280, 100)])
@pytest.mark.parametrize("abs_scale,crosscheck,tuple_test,tuple_scale", FLAG_CASES)
def test_restatement_equals_oracle(ns, nd, nc, abs_scale, crosscheck, tuple_test, tuple_scale):
    mp = synth.matcher_problem(ns, nd, nc, seed=ns + 3 * nd + nc)
    args = (mp["src_pts"], mp["dst_pts"], mp["src_feat"], mp["dst_feat"], abs_scale, crosscheck, tuple_test,
            tuple_scale)
    want, go = orc.match_correspondences(*args, tuple_seed=42, return_scale=True)
    got, g = mr.match(*args, tuple_seed=42)
    assert np.array_equal(got, want)
    assert g.tobytes() == F32(go).tobytes()


@pytest.mark.parametrize("kind", ["nan_src", "nan_both", "pinf", "minf", "coincident"])
@pytest.mark.parametrize("abs_scale,tuple_test", [(False, False), (False, True), (True, True)])
def test_restatement_equals_oracle_on_nonfinite_points(kind, abs_scale, tuple_test):
    sp, tp, _, _, sf, tf = mr.nonfinite_case(kind)
    args = (sp, tp, sf, tf, abs_scale, not tuple_test, tuple_test, 0.95)
    want, go = orc.match_correspondences(*args, tuple_seed=7, return_scale=True)
    got, g = mr.match(*args, tuple_seed=7)
    assert np.array_equal(got, want)
    assert g.tobytes() == F32(go).tobytes()


def test_accumulate_is_a_sequential_sum():
    rng = np.random.default_rng(1)
    for n in (1, 2, 3, 7, 8, 9, 31, 32, 33, 100):
        p = (1.0e4 + rng.uniform(-1, 1, size=(n, 3))).astype(F32)
        s = np.zeros(3, dtype=F32)
        for i in range(n):
            s = (s + p[i]).astype(F32)
        assert np.add.accumulate(p, axis=0, dtype=F32)[-1].tobytes() == s.tobytes()
        assert mr.sequential_mean(p).tobytes() == (s / F32(n)).astype(F32).tobytes()


def _splitmix_py(x):
    m = (1 << 64) - 1
    x = (x + 0x9E3779B97F4A7C15) & m
    x = ((x ^ (x >> 30)) * 0xBF58476D1CE4E5B9) & m
    x = ((x ^ (x >> 27)) * 0x94D049BB133111EB) & m
    return x ^ (x >> 31)


@pytest.mark.parametrize("seed", [0, 1, 2**63, 2**64 - 1, 2**64 - 2])
def test_draws_wrap_like_uint64(seed):
    r = mr.draws(seed, 7)
    for t in range(0, 700, 37):
        for k in range(3):
            assert r[t, k] == (_splitmix_py((seed + 3 * t + k) & ((1 << 64) - 1)) >> 33) % 7


@pytest.mark.parametrize("n", [31, 32, 33, 63, 64, 65, 1000, 20000, 100003])
def test_offset_clouds_scale_follows_the_summation_order(n):
    src, dst, _, _ = mr.offset_clouds(n, mr.offset_seed(n))
    g = mr.global_scale(src, dst)
    assert g == mr.max_scale(src, mr.sequential_mean(src)) > mr.max_scale(dst, mr.sequential_mean(dst))
    for mean in (mr.pairwise_mean, mr.float64_mean, mr.lane_strided_mean):
        assert mr.global_scale(src, dst, mean=mean).tobytes() != g.tobytes(), mean.__name__


def test_offset_clouds_of_one_point_take_the_target_scale():
    src, dst, _, _ = mr.offset_clouds(1, mr.offset_seed(1))
    assert mr.global_scale(src, dst) == mr.max_scale(dst, mr.sequential_mean(dst)) > 0


def test_nonfinite_scales():
    sp, tp, cs, ct, _, _ = mr.nonfinite_case("nan_src")
    g = mr.global_scale(sp, tp)
    assert g == mr.max_scale(tp, mr.sequential_mean(tp)) > 0
    assert g != mr.global_scale(cs, ct)
    assert np.isnan(mr.sequential_mean(sp)[1])
    assert mr.global_scale(*mr.nonfinite_case("nan_both")[:2]) == 0
    assert mr.global_scale(*mr.nonfinite_case("pinf")[:2]) == np.inf
    assert mr.global_scale(*mr.nonfinite_case("minf")[:2]) == np.inf
    assert mr.global_scale(*mr.nonfinite_case("coincident")[:2]) == 0


def test_coincident_points_keep_nothing_in_the_tuple_test():
    sp, tp, _, _, sf, tf = mr.nonfinite_case("coincident")
    assert len(mr.match(sp, tp, sf, tf, False, False, False, 0.0)[0]) > 0
    assert len(mr.match(sp, tp, sf, tf, False, False, True, 0.95)[0]) == 0


def _edge_lengths(s):
    lo, hi = F32(10.0) * F32(s), F32(10.0) / F32(s)
    up, dn = F32(np.inf), F32(-np.inf)
    return [(lo, False), (np.nextafter(lo, up), True), (np.nextafter(lo, dn), False),
            (hi, False), (np.nextafter(hi, dn), True), (np.nextafter(hi, up), False)]


@pytest.mark.parametrize("s", [0.5, 0.25])
def test_triangles_put_one_side_on_the_bound(s):
    for lj, inside in _edge_lengths(s):
        src, dst, sf, tf = mr.triangle_pair(lj)
        assert mr.sequential_mean(src).tolist() == [0, 0, 0] and mr.sequential_mean(dst).tolist() == [0, 0, 0]
        tr = mr.tuple_trials(src, dst, sf, tf, True, True, s, 0)
        assert tr["corres"].tolist() == [[0, 0], [1, 1], [2, 2]]
        perm = [tuple(r) for r in tr["r"]]
        assert set(itertools.permutations(range(3))) <= set(perm)          # every order of the triple is drawn
        for t, r in enumerate(perm):
            if len(set(r)) < 3:
                assert not tr["passed"][t]
                continue
            e_ab = [e for e, (u, v) in enumerate(((0, 1), (1, 2), (2, 0))) if {r[u], r[v]} == {0, 1}][0]
            assert tr["li"][t, e_ab] == 10 and tr["lj"][t, e_ab] == F32(lj)
            others = [e for e in range(3) if e != e_ab]
            li, lj_ = tr["li"][t, others], tr["lj"][t, others]
            assert np.all((li * F32(s) < lj_) & (lj_ < li / F32(s)))             # the AB side alone decides
            assert tr["passed"][t] == inside


@pytest.mark.parametrize("k", [6, 10])
def test_last_pair_is_present(k):
    for ns in (2**k - 1, 2**k, 2**k + 1):
        for nd in (2**k - 1, 2**k, 2**k + 1):
            for cc in (False, True):
                pairs, _ = mr.match(*mr.last_pair_case(ns, nd, seed=ns + nd), False, cc, False, 0.0)
                assert [ns - 1, nd - 1] in pairs.tolist()


def test_hub_has_one_hit():
    src, dst, sf, tf = mr.hub_case()
    swapped, corres, hit = mr.correspondences(len(src), len(dst), sf, tf, False)
    assert not swapped and np.flatnonzero(hit).tolist() == [123]
    assert len(corres) == 1 + len(dst)


def test_duplicates_tie():
    src, dst, sf, tf = mr.duplicate_case()
    assert mr.tie_count(tf, sf) == len(tf) and mr.tie_count(sf, tf) > 0
    _, corres, hit = mr.correspondences(len(src), len(dst), sf, tf, True)
    assert np.flatnonzero(hit).max() < 700 and len(corres) == hit.sum()   # the first copies win every tie


def test_strange_tuple_scales_keep_nothing():
    mp = synth.matcher_problem(300, 250, 120, seed=9)
    args = (mp["src_pts"], mp["dst_pts"], mp["src_feat"], mp["dst_feat"], False, False, True)
    assert len(mr.match(*args, 0.5, 3)[0]) > 0
    for s in (1.0, 1.05, -0.5, float("nan")):
        assert len(mr.match(*args, s, 3)[0]) == 0
