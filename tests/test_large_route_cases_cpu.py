"""The premises of tests/test_gpu_large_route_boundary.py, checked without a GPU: each case's exact core, its clique
number, that the device's capped peels would stop on a superset above the cap they are meant to cross, and that the
greedy's top-degree root lies in the planted clique, so the incumbent L is the one the GPU test expects."""
import numpy as np
import pytest

import large_route_cases as C
import oracle_lib as orc

IN_PLACE_ROUNDS = 48      # kCoreRounds: one launch each on the large route
LAYERED_ROUNDS = 256      # the small route's former peel cap
CAP, CAP64 = 32768, 64


def _top_root_in_clique(case):
    deg = C.degrees(case["n"], case["edges"])
    root = int(np.argmax(deg))  # the largest degree, the lowest index among ties: the greedy's first root
    assert root in set(case["clique"].tolist()) and deg[root] > np.delete(deg, case["clique"]).max(initial=0)


def _oracle_clique(case):
    c, info = orc.max_clique_bits(C.to_bits(case["n"], case["edges"]), case["n"])
    assert not info["timed_out"]
    return c


def test_bits_round_trip():
    case = C.slow_peel_case("several")
    bits = C.to_bits(case["n"], case["edges"])
    assert np.array_equal(C.edges_of_bits(bits, case["n"]), case["edges"])
    assert bits.shape == (4096, 64) and int(C.degrees(4096, case["edges"]).sum()) == 2 * len(case["edges"])


def test_core_numbers_and_peel_on_hand_cases():
    # a K4 with a pendant triangle path: core numbers 3, 3, 3, 3 | 1, 1, 1
    e = C.clique_edges([0, 1, 2, 3]).tolist() + [[3, 4], [4, 5], [5, 6]]
    assert C.core_numbers(7, e).tolist() == [3, 3, 3, 3, 1, 1, 1]
    assert C.kcore(7, e, 3).tolist() == [0, 1, 2, 3] and C.kcore(7, e, 4).size == 0
    # the layered peel of a path of 5 hanging from a triangle: the end goes at the start, then one per round
    case = C.pendant_paths(8, [0, 1, 2], [(3, 5)])
    for r in range(6):
        alive, _ = C.layered_peel(8, case["edges"], 2, rounds=r)
        assert len(alive) == C.layered_survivors_bound(3, [5], r)


@pytest.mark.parametrize("name", ["one300", "lp260", "several", "paths250"])
def test_slow_peel_premises(name):
    case = C.slow_peel_case(name)
    n, e = case["n"], case["edges"]
    assert np.array_equal(C.kcore(n, e, 2), case["clique"]) and len(case["clique"]) == 3
    assert np.array_equal(C.innermost_core(n, e), case["clique"])
    # trees on a triangle: the clique number is 3 and the triangle is the only triangle
    assert len(e) == 3 + sum(case["paths"])
    _top_root_in_clique(case)
    # the layered bound is what layered peeling leaves
    for r in (0, 1, 100, LAYERED_ROUNDS):
        assert len(C.layered_peel(n, e, 2, rounds=r)[0]) == C.layered_survivors_bound(3, case["paths"], r)
    inplace = C.inplace_survivors_bound(3, case["paths"], IN_PLACE_ROUNDS)
    layered = C.layered_survivors_bound(3, case["paths"], LAYERED_ROUNDS)
    # 48 in-place rounds stop on a superset above the test cap; 256 layered rounds (small route: n <= 32768 only)
    # stop on more than the core
    assert inplace > CAP64 and (layered > 3 or n > CAP)
    if name == "paths250":
        assert inplace > CAP  # the large route would give up on a graph whose core is a triangle
    if name == "lp260":
        assert layered == 6  # 2L >= |alive|: the LP kernel runs on this superset instead of giving up
    if name == "several":
        assert layered > 4 * 3 + 64  # the second chance would run on the superset
    if n <= 4096:
        assert np.array_equal(_oracle_clique(case), case["clique"])


@pytest.mark.parametrize("size,n", [(63, 256), (64, 256), (65, 256), (32768, 65536), (32769, 65536)])
def test_cap_edge_premises(size, n):
    case = C.cap_case(size, n)
    e, L = case["edges"], case["L"]
    core = C.kcore(n, e, L - 1)
    assert len(core) == size and np.array_equal(core, case["core"])
    assert np.array_equal(C.layered_peel(n, e, L - 1, rounds=1)[0], core)  # converges at the start
    _top_root_in_clique(case)
    if n <= 4096:
        assert np.array_equal(_oracle_clique(case), case["clique"])
    rounds, S = C.second_chance_rounds(n, e, core, L)
    assert rounds <= 3 and np.array_equal(S, case["clique"])
    assert (size <= CAP64) == (size in (63, 64)) and (size <= CAP) == (size != 32769 and size <= 32768)


@pytest.mark.parametrize("n", [4096, 65536])
def test_word_edge_premises(n):
    case = C.word_edge_case(n)
    e, L, cl = case["edges"], case["L"], case["clique"]
    core = C.kcore(n, e, L - 1)
    assert np.array_equal(core, case["core"]) and len(core) == 1537
    pos = np.searchsorted(core, cl)
    assert pos.tolist() == [31, 32, 63, 64, 1023, 1024, 1536] and cl[-1] == n - 1
    if n == 65536:
        assert np.all(np.isin(core % 32, [0, 31])) and {0, 31, 32767, 32768}.issubset(set(core.tolist()))
    else:
        assert {0, 31, 32, 63, 1023, 1024, 2047, 2048}.issubset(set(core.tolist()))
        assert np.array_equal(_oracle_clique(case), cl)
    _top_root_in_clique(case)
    rounds, S = C.second_chance_rounds(n, e, core, L)
    assert rounds <= 3 and np.array_equal(S, cl)


def test_mixed_batch_premises():
    cases = C.mixed_batch_cases()
    assert [c["n"] for _, c, _ in cases] == [36000] * len(cases)
    for name, case, route in cases:
        n, e, L = case["n"], case["edges"], case["L"]
        if name == "edgeless":
            assert len(e) == 0 and route == 1
            continue
        core = C.kcore(n, e, L - 1)
        assert np.array_equal(core, case["core"]), name
        _top_root_in_clique(case)
        if name == "above_cap":
            assert route == -1 and len(core) > CAP
        elif name == "slow":
            assert route == 3 and C.inplace_survivors_bound(3, case["paths"], IN_PLACE_ROUNDS) > 700
        else:
            assert route == len(core) <= CAP, name
    sizes = sorted(r for _, _, r in cases if r > 8)
    assert sizes == [200, 1200]  # searched cores of two sizes: the smaller one is padded to 1200


def test_two_motion_scene_premises():
    sc = C.two_motion_scene(40000, 24, 4)
    n, m = sc["n"], sc["m"]
    union = np.sort(np.concatenate(sc["groups"]))
    core = C.kcore(n, sc["edges"], m - 1)
    assert np.array_equal(core, union)  # the route compacts and searches 2m vertices
    assert sc["margin"] > 1e-6          # no pair within rounding of the threshold
    # every clique of size >= m lies in the (m-1)-core: the exact answer on the core's induced graph is the answer
    sub = np.isin(sc["edges"], union).all(1)
    local = np.searchsorted(union, sc["edges"][sub])
    c, info = orc.max_clique_bits(C.to_bits(2 * m, local), 2 * m)
    assert not info["timed_out"] and np.array_equal(union[c], sc["expect"])
    assert len(sc["expect"]) == m and sc["expect"][0] < min(g[0] for g in sc["groups"] if g is not sc["expect"])
