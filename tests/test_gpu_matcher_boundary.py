"""The correspondence stage where it can be wrong (csrc/matcher.cu; DESIGN.md 3.8), on the device against the numpy
restatement tests/matcher_reference.py, bit for bit: the pairs and the float32 bytes of global_scale_.  Every test
first asserts its premise (the tests/test_matcher_reference_cpu.py checks hold the same ones on the CPU), so none
can pass vacuously.

* mean_kernel's single sequential sum: clouds at 1e4 whose scale changes under any other summation order, across
  the kernel's 32-point lookahead.
* Non-finite and degenerate points: NaN drops a cloud from the scale, inf makes it inf, coincident clouds give 0.
* center_kernel's warp-uniform reduction: batches whose pair boundaries fall inside warps, a poisoned pair among them.
* The tuple test's six strict bounds at equality and one ulp either side; degenerate triples; odd tuple scales.
* Trial dealing over several grid strides; seeds whose draws wrap 2^64.
* Key packing: the correspondence (ns - 1, nd - 1) at power-of-two sizes, alone and in batches.
* The larger cloud is "i" (strictly), the hit rule, mutual ties, and the 1024-slot compaction loops."""
import importlib

import numpy as np
import pytest

import matcher_reference as mr
import oracle_lib as orc

capi = importlib.import_module("teaser-plusplus_b200.capi")
synth = importlib.import_module("teaser-plusplus_b200.synth")

pytestmark = pytest.mark.gpu
F32 = np.float32

FLAG_CASES = [(abs_s, cc, tt, ts) for abs_s in (False, True) for cc in (False, True)
              for (tt, ts) in ((False, 0.0), (True, 0.95), (True, 0.0), (False, 0.95))]


@pytest.fixture(scope="module")
def ctx():
    c = capi.Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def stride():
    """tuple_kernel's grid stride: 8 CTAs of 256 threads per SM."""
    import torch
    return 8 * torch.cuda.get_device_properties(0).multi_processor_count * 256


def _same(got, g, want, gw):
    return np.array_equal(got, want) and F32(g).tobytes() == F32(gw).tobytes()


def _check(ctx, case, flags, seed=0, oracle=False):
    """One pair on the device == the restatement (and the oracle); returns the restatement's pairs and scale."""
    want, gw = mr.match(*case, *flags, tuple_seed=seed)
    got, g = ctx.match_correspondences(*case, *flags, tuple_seed=seed, return_scale=True)
    assert np.array_equal(got, want)
    assert F32(g).tobytes() == gw.tobytes()
    if oracle:
        wo, go = orc.match_correspondences(*case, *flags, tuple_seed=seed, return_scale=True)
        assert _same(wo, go, want, gw)
    return want, gw


def _check_batch(ctx, cases, flags, seeds, wants=None):
    """The batch entry == every pair's restatement (given or computed) and its single call."""
    wants = wants or [mr.match(*c, *flags, tuple_seed=s) for c, s in zip(cases, seeds)]
    got, gs = ctx.match_correspondences_batch(*zip(*cases), *flags, tuple_seeds=seeds, return_scale=True)
    for b, (c, s, (w, gw)) in enumerate(zip(cases, seeds, wants)):
        assert np.array_equal(got[b], w), b
        assert F32(gs[b]).tobytes() == gw.tobytes(), b
        one, g1 = ctx.match_correspondences(*c, *flags, tuple_seed=s, return_scale=True)
        assert _same(one, g1, w, gw), b
    return wants


# ---- the sequential mean ---------------------------------------------------------------------------------------------
MEAN_SIZES = [1, 31, 32, 33, 63, 64, 65, 1000, 20000, 100003]
MEAN_FLAGS = [(False, True, False, 0.0), (False, False, True, 0.9)]


@pytest.fixture(scope="module")
def offset_cases():
    cases = {}
    for n in MEAN_SIZES:
        src, dst, sf, tf = mr.offset_clouds(n, mr.offset_seed(n))
        g = mr.global_scale(src, dst)
        if n >= 31:   # premise: any other summation order changes the scale's bits
            for mean in (mr.pairwise_mean, mr.float64_mean, mr.lane_strided_mean):
                assert mr.global_scale(src, dst, mean=mean).tobytes() != g.tobytes(), (n, mean.__name__)
        else:         # one source point: its mean is the point; the target sets the scale
            assert g == mr.max_scale(dst, mr.sequential_mean(dst)) > 0
        cases[n] = (src, dst, sf, tf)
    return cases


@pytest.mark.parametrize("n", MEAN_SIZES)
@pytest.mark.parametrize("flags", MEAN_FLAGS)
def test_sequential_mean(ctx, offset_cases, n, flags):
    _check(ctx, offset_cases[n], flags, seed=5, oracle=n >= 20000)


@pytest.mark.parametrize("flags", MEAN_FLAGS)
def test_sequential_mean_batch(ctx, offset_cases, flags):
    cases = [offset_cases[n] for n in MEAN_SIZES]
    _check_batch(ctx, cases, flags, [5] * len(cases))
    _check_batch(ctx, cases[::-1], flags, [5] * len(cases))


# ---- non-finite and degenerate points --------------------------------------------------------------------------------
KINDS = ["nan_src", "nan_both", "pinf", "minf", "coincident"]


def _expected_scale(kind, sp, tp):
    return {"nan_src": mr.max_scale(tp, mr.sequential_mean(tp)), "nan_both": F32(0), "pinf": F32(np.inf),
            "minf": F32(np.inf), "coincident": F32(0)}[kind]


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("abs_scale", [False, True])
@pytest.mark.parametrize("tuple_test", [False, True])
def test_nonfinite_points(ctx, kind, abs_scale, tuple_test):
    sp, tp, cs, ct, sf, tf = mr.nonfinite_case(kind)
    flags = (abs_scale, not tuple_test, tuple_test, 0.95)
    want, g = _check(ctx, (sp, tp, sf, tf), flags, seed=7)
    if abs_scale:
        assert g == F32(1.0)
    else:
        assert g.tobytes() == _expected_scale(kind, sp, tp).tobytes()
        if kind == "nan_src":   # premise: the clean source would have set the scale
            assert mr.global_scale(cs, ct) > g > 0
    if not tuple_test:          # the pairs follow the descriptors alone
        clean, _ = mr.match(cs, ct, sf, tf, *flags)
        assert np.array_equal(want, clean) and len(want) > 0
    elif kind == "coincident" and not abs_scale:
        assert len(want) == 0   # every normalised point is 0 / 0: no triple passes


# ---- batches whose pair boundaries fall inside warps -----------------------------------------------------------------
WARP_SIZES = [(1, 5), (5, 31), (31, 33), (33, 37), (37, 1), (33, 33), (5, 5), (37, 31)]


@pytest.fixture(scope="module")
def warp_cases():
    cases = []
    for b, (ns, nd) in enumerate(WARP_SIZES):
        mp = synth.matcher_problem(ns, nd, min(ns, nd) // 2, seed=100 + b)
        k = F32(2.0 ** (b - 3))      # every pair its own spread, so a scale given to the wrong pair shows
        cases.append(((mp["src_pts"] * k).astype(F32), (mp["dst_pts"] * k).astype(F32), mp["src_feat"],
                      mp["dst_feat"]))
    sp, tp, _, _, sf, tf = mr.nonfinite_case("nan_src")
    poisoned = (sp[:33], tp[:31], sf[:33], tf[:31])
    cases.insert(3, poisoned)
    gs = [mr.global_scale(c[0], c[1]) for c in cases]
    assert len(set(g.tobytes() for g in gs)) == len(gs)           # premise: the scales are pairwise distinct
    assert np.isnan(mr.sequential_mean(poisoned[0])).any()
    return cases


@pytest.mark.parametrize("order", ["forward", "reversed"])
@pytest.mark.parametrize("flags", [(False, False, False, 0.0), (False, True, True, 0.9)])
def test_pair_boundaries_inside_warps(ctx, warp_cases, order, flags):
    cases = warp_cases if order == "forward" else warp_cases[::-1]
    _check_batch(ctx, cases, flags, list(range(len(cases))))


# ---- the tuple test's strict bounds ----------------------------------------------------------------------------------
def _edge_lengths(s):
    lo, hi = F32(10.0) * F32(s), F32(10.0) / F32(s)
    up, dn = F32(np.inf), F32(-np.inf)
    return [("lower", lo, False), ("lower+1ulp", np.nextafter(lo, up), True),
            ("lower-1ulp", np.nextafter(lo, dn), False), ("upper", hi, False),
            ("upper-1ulp", np.nextafter(hi, dn), True), ("upper+1ulp", np.nextafter(hi, up), False)]


@pytest.mark.parametrize("s", [0.5, 0.25])
@pytest.mark.parametrize("edge", range(6))
@pytest.mark.parametrize("crosscheck", [True, False])
def test_tuple_bounds_are_strict(ctx, s, edge, crosscheck):
    name, lj, inside = _edge_lengths(s)[edge]
    case = mr.triangle_pair(lj)
    tr = mr.tuple_trials(*case, True, crosscheck, s, 0)
    # premise: |AB| is li = 10 against lj exactly, both other sides are strictly inside, and every order of the
    # three correspondences is drawn, so AB stands in each of the six comparisons
    drawn = {tuple(tr["corres"][r].reshape(-1)) for r in tr["r"] if len({tuple(tr["corres"][x]) for x in r}) == 3}
    assert len(drawn) == 6, name
    distinct = np.array([len({tuple(tr["corres"][x]) for x in r}) == 3 for r in tr["r"]])
    assert np.all(tr["passed"][distinct] == inside) and not tr["passed"][~distinct].any(), name
    want, _ = _check(ctx, case, (True, crosscheck, True, s))
    assert want.tolist() == ([[0, 0], [1, 1], [2, 2]] if inside else []), name


@pytest.mark.parametrize("n", [1, 2])
@pytest.mark.parametrize("crosscheck", [True, False])
def test_degenerate_triples(ctx, n, crosscheck):
    src, dst, sf, tf = mr.triangle_pair(10.0)
    case = (src[:n], dst[:n], sf[:n], tf[:n])
    tr = mr.tuple_trials(*case, True, crosscheck, 0.5, 0)
    assert len({tuple(c) for c in tr["corres"]}) == n and len(tr["r"]) > 0     # premise: only repeated triples
    want, _ = _check(ctx, case, (True, crosscheck, True, 0.5))
    assert len(want) == 0
    assert len(_check(ctx, case, (True, crosscheck, False, 0.5))[0]) == n


@pytest.mark.parametrize("s", [1.0, 1.05, -0.5, float("nan")])
def test_tuple_scales_that_keep_nothing(ctx, s):
    mp = synth.matcher_problem(300, 250, 120, seed=9)
    case = (mp["src_pts"], mp["dst_pts"], mp["src_feat"], mp["dst_feat"])
    assert len(_check(ctx, case, (False, False, True, 0.5), seed=3)[0]) > 0     # premise: the test keeps at 0.5
    assert len(_check(ctx, case, (False, False, True, s), seed=3)[0]) == 0


# ---- trial dealing ---------------------------------------------------------------------------------------------------
DEAL_SEEDS = [0, 2**63, 2**64 - 1, 2**64 - 2, 1, 2**63 - 1, 2**40 + 17, 12345, 2**64 - 150]


def test_trials_wrap_the_grid_stride(ctx, stride):
    cases, ncorr = [], 0
    for b, seed in enumerate(DEAL_SEEDS):
        mp = synth.matcher_problem(1300 - 37 * b, 1100 + 23 * b, 500, seed=200 + b, feat_noise=0.3)
        case = (mp["src_pts"], mp["dst_pts"], mp["src_feat"], mp["dst_feat"])
        cases.append(case)
        ncorr += len(mr.correspondences(len(case[0]), len(case[1]), case[2], case[3], False)[1])
    assert 100 * ncorr > 4 * stride                                           # premise: the trials wrap 4+ times
    flags = (False, False, True, 0.9)
    wants = _check_batch(ctx, cases, flags, DEAL_SEEDS)
    for c, s, (w, _) in zip(cases, DEAL_SEEDS, wants):                        # premise: the draws matter
        assert 0 < len(w) and not np.array_equal(w, mr.match(*c, *flags, tuple_seed=s ^ 1)[0])
    _check_batch(ctx, cases[::-1], flags, DEAL_SEEDS[::-1], wants[::-1])
    _check(ctx, cases[2], flags, seed=DEAL_SEEDS[2], oracle=True)


# ---- key packing -----------------------------------------------------------------------------------------------------
PACK_SIZES = [(ns, nd) for k in (6, 10) for ns in (2**k - 1, 2**k, 2**k + 1) for nd in (2**k - 1, 2**k, 2**k + 1)]


@pytest.mark.parametrize("ns,nd", PACK_SIZES)
@pytest.mark.parametrize("crosscheck", [True, False])
def test_last_pair_survives_key_packing(ctx, ns, nd, crosscheck):
    want, _ = _check(ctx, mr.last_pair_case(ns, nd, seed=ns + nd), (False, crosscheck, False, 0.0))
    assert [ns - 1, nd - 1] in want.tolist()


SMALL = [(37, 20), (5, 9), (64, 64), (1, 1), (200, 130), (9, 5), (33, 31), (2, 3)]


@pytest.mark.parametrize("B", [1, 2, 3, 4, 5, 8, 9])
def test_batch_pair_bits(ctx, B):
    big = mr.last_pair_case(1024, 1024, seed=2048)
    cases = [mr.last_pair_case(ns, nd, seed=ns * 7 + nd) for ns, nd in SMALL[:B - 1]]
    cases.insert(B // 2, big)
    flags = (False, True, False, 0.0)
    wants = _check_batch(ctx, cases, flags, [0] * B)
    assert [1023, 1023] in wants[B // 2][0].tolist()
    for c, (w, _) in zip(cases, wants):
        assert [len(c[0]) - 1, len(c[1]) - 1] in w.tolist()


# ---- which cloud is "i" ----------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def mirror_cases():
    out = {}
    for ns, nd in [(300, 257), (257, 300), (1025, 1024), (300, 300), (301, 300), (300, 301)]:
        mp = synth.matcher_problem(ns, nd, 120, seed=ns * 3 + nd, feat_noise=0.3)
        out[(ns, nd)] = (mp["src_pts"], mp["dst_pts"], mp["src_feat"], mp["dst_feat"])
    return out


def _mirror(ctx, case, flags, seed):
    sp, tp, sf, tf = case
    got, g = ctx.match_correspondences(tp, sp, tf, sf, *flags, tuple_seed=seed, return_scale=True)
    got = got[:, ::-1]
    return got[np.lexsort((got[:, 1], got[:, 0]))], g


@pytest.mark.parametrize("sizes", [(300, 257), (257, 300), (1025, 1024)])
@pytest.mark.parametrize("abs_scale,crosscheck,tuple_test,tuple_scale", FLAG_CASES)
def test_mirror_with_unequal_sizes(ctx, mirror_cases, sizes, abs_scale, crosscheck, tuple_test, tuple_scale):
    flags = (abs_scale, crosscheck, tuple_test, tuple_scale)
    want, gw = _check(ctx, mirror_cases[sizes], flags, seed=17)
    got, g = _mirror(ctx, mirror_cases[sizes], flags, 17)
    assert np.array_equal(got, want) and F32(g).tobytes() == gw.tobytes()


@pytest.mark.parametrize("sizes", [(300, 300), (301, 300), (300, 301)])
@pytest.mark.parametrize("abs_scale,crosscheck,tuple_test,tuple_scale", FLAG_CASES)
def test_equal_and_adjacent_sizes(ctx, mirror_cases, sizes, abs_scale, crosscheck, tuple_test, tuple_scale):
    flags = (abs_scale, crosscheck, tuple_test, tuple_scale)
    want, _ = _check(ctx, mirror_cases[sizes], flags, seed=17)
    if sizes == (300, 300) and not crosscheck and not (tuple_test and tuple_scale):
        # at ns == nd the source stays "i", so the mirrored call lists other correspondences
        sp, tp, sf, tf = mirror_cases[sizes]
        mw = mr.match(tp, sp, tf, sf, *flags, tuple_seed=17)[0][:, ::-1]
        mw = mw[np.lexsort((mw[:, 1], mw[:, 0]))]
        assert not np.array_equal(mw, want)                                  # premise
        assert np.array_equal(_mirror(ctx, mirror_cases[sizes], flags, 17)[0], mw)


# ---- hit rule, mutual ties, compaction -------------------------------------------------------------------------------
@pytest.mark.parametrize("crosscheck", [True, False])
@pytest.mark.parametrize("mirrored", [False, True])
def test_hub_is_the_only_hit(ctx, crosscheck, mirrored):
    src, dst, sf, tf = mr.hub_case()
    _, corres, hit = mr.correspondences(len(src), len(dst), sf, tf, crosscheck)
    assert np.flatnonzero(hit).tolist() == [123]                             # premise
    case = (dst, src, tf, sf) if mirrored else (src, dst, sf, tf)
    want, _ = _check(ctx, case, (False, crosscheck, False, 0.0))
    hub_col = want[:, 1] if mirrored else want[:, 0]
    assert set(hub_col.tolist()) == {123} and len(want) == (1 if crosscheck else len(dst))


@pytest.mark.parametrize("crosscheck", [True, False])
@pytest.mark.parametrize("tuple_test", [False, True])
def test_duplicates_across_segments(ctx, crosscheck, tuple_test):
    case = mr.duplicate_case()
    src, dst, sf, tf = case
    assert mr.tie_count(tf, sf) == len(tf)                                   # premise: every target ties
    want, _ = _check(ctx, case, (False, crosscheck, tuple_test, 0.9), seed=4)
    assert len(want) > 0


SLOTS = [1023, 1024, 1025, 2047, 2048, 2049]


@pytest.mark.parametrize("slots", SLOTS)
@pytest.mark.parametrize("crosscheck", [True, False])
def test_compaction_slot_counts(ctx, slots, crosscheck):
    ns, nd = (slots, slots - 300) if crosscheck else (slots - slots // 2, slots // 2)
    mp = synth.matcher_problem(ns, nd, min(ns, nd) // 2, seed=slots, feat_noise=0.2)
    case = (mp["src_pts"], mp["dst_pts"], mp["src_feat"], mp["dst_feat"])
    _, corres, _ = mr.correspondences(ns, nd, case[2], case[3], crosscheck)
    # premise: valid slots run up to the last 1024-slot chunk (slot i for the cross check, n_i + j without it)
    assert corres[:, 0].max() >= slots - 64 if crosscheck else len(corres) > slots - 1024
    _check(ctx, case, (False, crosscheck, False, 0.0))
    _check(ctx, case, (False, crosscheck, True, 0.9), seed=slots)
