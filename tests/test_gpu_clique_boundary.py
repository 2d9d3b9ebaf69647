"""The exact max-clique stage where it can be wrong (run on an H100: `pytest -m gpu`).

Every result is checked to be a clique and compared with a reference that does not share the kernel's code: a closed
form (complete multipartite graphs, cocktail-party graphs, complements of triangles and stars, two-motion scenes) or
the CPU oracle (`orc.max_clique_bits`, `orc.solve`).  The parity contract is the identical sorted index set, so among
tied maximum cliques the lexicographically smallest one.

What is covered: many tied maxima recorded concurrently by different warps; clique members at bitset word edges
(v % 32 in {0, 31}, n - 1) and n on both sides of 32, 64, 128, 1024; the second-chance heuristic and the singleton-class
A/B switch (debug flag 8192); the batched exact search (`tzr_max_clique_batch`: start groups, scratch moving between
problems, per-problem strict mode, deadline and counters); the three outcomes after the first pass, made independent of
machine load by debug flag 32768 (1 ns first pass); strict mode that must not follow a warp into the next problem;
tie enumeration made independent of the 50 ms first pass by debug flag 131072 (one pass); the depth cap, made reachable by debug flag 65536 (8 levels); the
input contract (diagonal and out-of-range bits ignored); and ties inside the whole solve path, single and batched.
"""
import importlib

import numpy as np
import pytest

import oracle_lib as orc

capi = importlib.import_module("teaser-plusplus_b200.capi")
synth = importlib.import_module("teaser-plusplus_b200.synth")

pytestmark = pytest.mark.gpu

FLAG_NO_SINGLES = 8192       # exact search without the singleton-class path of the colouring (same output)
FLAG_SHORT_FIRST = 32768     # first exact pass of 1 ns: every open problem goes through the LP kernel
FLAG_DEPTH8 = 65536          # exact-search stack of 8 levels
FLAG_ONE_PASS = 131072       # one exact pass with the whole budget: no 50 ms cap, no LP kernel
ROT_TOL = 1e-4   # rad, as tests/test_gpu_parity.py
TRANS_TOL = 1e-4  # m
# Tied maxima are enumerated serially under their smallest vertex (one warp per root), about 10-20 us per search
# node: 2^14 ties overrun the 50 ms first pass (the LP bound then closes the problem, proven = 2).  The tie tests run
# under FLAG_ONE_PASS, so their outcome does not depend on the wall clock; tie problems searched with the default
# two passes keep SMALL_TIES, a few hundred microseconds of enumeration.
MAX_TIES = 1 << 12
SMALL_TIES = 1 << 5


@pytest.fixture(scope="module")
def ctx():
    c = capi.Context(0)
    yield c
    c.close()


@pytest.fixture()
def flags(ctx):
    """Set debug flags for one test; always cleared afterwards."""
    yield ctx.set_flags
    ctx.set_flags(0)


# ------------------------------------------------------------------ graph construction (numpy only)
def bits_of(A):
    n = A.shape[0]
    W = (n + 63) // 64
    padded = np.zeros((n, W * 64), dtype=np.uint8)
    padded[:, :n] = A
    return np.packbits(padded, axis=1, bitorder="little").view(np.uint64).reshape(n, W)


def sym(U):
    U = np.triu(U, 1)
    return U | U.T


def gnp(n, p, rng):
    return sym(rng.uniform(size=(n, n)) < p)


def plant(A, members):
    m = np.asarray(sorted(members))
    A[np.ix_(m, m)] = True
    np.fill_diagonal(A, False)
    return A


def assert_clique(A, c):
    c = np.asarray(c)
    assert np.all(np.diff(c) > 0), "not sorted / not unique"
    assert c.size == 0 or (c[0] >= 0 and c[-1] < A.shape[0])
    sub = A[np.ix_(c, c)]
    assert sub.sum() == c.size * (c.size - 1), "not a clique"


def multipartite(n, sizes, rng, minima=()):
    """Complete multipartite graph: vertices are adjacent iff they lie in different parts.  Part j < len(minima) has
    smallest label minima[j]; everything else is labelled at random.  Every transversal is a maximum clique, so
    omega = number of parts, there are prod(sizes) ties, and the canonical answer is {min of each part}."""
    assert sum(sizes) == n
    part = np.full(n, -1)
    free = np.ones(n, dtype=bool)
    for j, m in enumerate(minima):
        part[m] = j
        free[m] = False
    for j in sorted(range(len(minima)), key=lambda j: -minima[j]):  # most constrained first
        cand = np.nonzero(free & (np.arange(n) > minima[j]))[0]
        pick = rng.choice(cand, sizes[j] - 1, replace=False)
        part[pick] = j
        free[pick] = False
    rest = rng.permutation(np.nonzero(free)[0])
    pos = 0
    for j in range(len(minima), len(sizes)):
        part[rest[pos:pos + sizes[j]]] = j
        pos += sizes[j]
    A = part[:, None] != part[None, :]
    canon = np.array(sorted(int(np.nonzero(part == j)[0].min()) for j in range(len(sizes))), dtype=np.int32)
    return A, canon


def tie_graph(n, rng, word_edges=False, max_ties=MAX_TIES):
    """Multipartite graph with parts of 1 (universal vertices), 2 and 3 and at most max_ties tied maxima.  word_edges:
    part minima at v % 32 in {0, 31}, at the 1024-word edge and at n - 1."""
    minima, dsizes = [], []
    if word_edges:
        minima = sorted({m for m in (0, 31, 32, 63, 64, 95, 127, 128, 1023, 1024) if m < n - 1}) + [n - 1]
        dsizes = [2 if (i < 4 and m < n - 8) else 1 for i, m in enumerate(minima)]
    ties = int(np.prod(dsizes)) if dsizes else 1
    extra = []
    for s in rng.permutation([2, 2, 2, 2, 3, 3, 3, 2, 3, 2]):
        if sum(dsizes) + sum(extra) + s <= n and ties * s <= max_ties:
            extra.append(int(s))
            ties *= int(s)
    sizes = dsizes + extra + [1] * (n - sum(dsizes) - sum(extra))
    A, canon = multipartite(n, sizes, rng, minima)
    return A, canon, ties


def cocktail_party(pairs, rng):
    """Complement of a perfect matching: omega = pairs, 2^pairs ties; vertex-cover LP bound = pairs (tight)."""
    n = 2 * pairs
    perm = rng.permutation(n)
    A = ~np.eye(n, dtype=bool)
    a, b = perm[0::2], perm[1::2]
    A[a, b] = A[b, a] = False
    return A


def triangles_and_stars(T, leaves, rng):
    """Complement H of (T disjoint triangles + stars with the given leaf counts, each >= 2).  omega = T + S (one vertex
    per triangle, every leaf); the LP bound is n - ceil((3T + 2 stars) / 2), the star centres have LP value 1."""
    n = 3 * T + sum(leaves) + len(leaves)
    perm = rng.permutation(n)
    H = np.zeros((n, n), dtype=bool)
    v = 0
    for _ in range(T):
        t = perm[v:v + 3]
        v += 3
        for i in range(3):
            for j in range(3):
                H[t[i], t[j]] = i != j
    for s in leaves:
        assert s >= 2
        c, lv = perm[v], perm[v + 1:v + 1 + s]
        v += 1 + s
        H[c, lv] = H[lv, c] = True
    A = ~H
    np.fill_diagonal(A, False)
    omega = T + sum(leaves)
    lp_ub = n - (3 * T + 2 * len(leaves) + 1) // 2
    return A, omega, lp_ub


def word_edge_graph(n, rng):
    """Random graph with two planted cliques of equal size: one on indices 32k - 1, 32k and n - 1, one at random.  The
    planted size is a few above the random part's clique number, so the exact search runs over a large core."""
    p = 0.3 if n <= 129 else (0.1 if n <= 1025 else 0.05)
    size = 8 if n <= 129 else 9
    A = gnp(n, p, rng)
    edge = {n - 1}
    ks = [k for k in range(1, n // 32 + 1) if 32 * k - 1 < n - 1]
    for k in rng.permutation(ks)[:3]:
        edge |= {32 * int(k) - 1} | ({32 * int(k)} if 32 * int(k) < n - 1 else set())
    others = rng.permutation(np.setdiff1d(np.arange(n), sorted(edge)))
    edge = sorted(edge | set(others[:max(0, size - len(edge))].tolist()))
    second = sorted(rng.choice(np.setdiff1d(np.arange(n), edge), size=len(edge), replace=False).tolist())
    plant(A, edge)
    plant(A, second)
    return A, edge


def second_chance_graph(n, p, k, rng):
    """G(n, p) plus a clique of k vertices at the top of the index range whose members keep the average degree (their
    other edges are thinned), so no top-degree root of the greedy heuristic belongs to it and the peel kernel's
    global-peeling second chance has to find it (alive > 4L + 64)."""
    A = gnp(n, p, rng)
    members = np.sort(rng.choice(np.arange(n - n // 10, n), size=k, replace=False))
    inside = np.zeros(n, dtype=bool)
    inside[members] = True
    keep = sym(rng.uniform(size=(n, n)) < (p * n - (k - 1)) / (p * n))
    A &= keep | ~(inside[:, None] | inside[None, :])
    plant(A, members)
    return A, members


def shortcut_graph(n, rng, k=12):
    """Sparse graph with one planted clique: only the clique survives its own core bound (the peel kernel's
    uniqueness shortcut, no exact search)."""
    A = gnp(n, 0.02, rng)
    members = rng.choice(n, size=k, replace=False)
    return plant(A, members), np.sort(members)


def oracle(A):
    c, info = orc.max_clique_bits(bits_of(A), A.shape[0])
    assert not info["timed_out"]
    return c


def single(ctx, A):
    """One problem through tzr_max_clique_batch (B = 1): (clique, proven code, search flags)."""
    cl, proven, f = ctx.max_clique_batch(bits_of(A)[None])
    return cl[0], int(proven[0]), int(f[0])


def check_proven(ctx, A, ref):
    gc, proven, _ = single(ctx, A)
    assert_clique(A, gc)
    assert proven == 1
    assert np.array_equal(gc, ref)
    return gc


# ------------------------------------------------------------------ tied maxima, closed form
TIE_NS = [31, 32, 33, 63, 64, 65, 127, 128, 129, 1023, 1024, 1025]


@pytest.mark.parametrize("word_edges", [False, True])
@pytest.mark.parametrize("n", TIE_NS)
def test_multipartite_ties_canonical(ctx, flags, n, word_edges):
    rng = np.random.default_rng(1000 + n + 7 * word_edges)
    A, canon, ties = tie_graph(n, rng, word_edges)
    assert ties <= MAX_TIES
    flags(FLAG_ONE_PASS)
    if word_edges:
        assert n - 1 in canon and 0 in canon
    gc, proven, f = single(ctx, A)
    assert_clique(A, gc)
    assert proven == 1 and f == 0, (proven, f)
    assert np.array_equal(gc, canon)
    g1, p1 = ctx.max_clique(bits_of(A), n, mode=0)
    assert p1 and np.array_equal(g1, canon)


# ------------------------------------------------------------------ word-edge placement vs the oracle
@pytest.mark.parametrize("n", [31, 32, 33, 63, 64, 65, 127, 128, 129, 1023, 1024, 1025, 4097])
def test_word_edge_cliques(ctx, n):
    rng = np.random.default_rng(2000 + n)
    A, edge = word_edge_graph(n, rng)
    ref = oracle(A)
    assert len(ref) >= len(edge)
    check_proven(ctx, A, ref)


# ------------------------------------------------------------------ search paths vs the oracle, with the A/B switch
def _search_case(name):
    rng = np.random.default_rng(sum(map(ord, name)))
    if name.startswith("gnp"):
        _, n, p = name.split("_")
        return gnp(int(n), float(p), rng)
    n = int(name.split("_")[1])
    A, _ = second_chance_graph(n, 0.15, n // 100, rng)
    return A


SEARCH_CASES = ["gnp_4000_0.05", "gnp_2000_0.1", "gnp_1000_0.2", "gnp_400_0.35", "gnp_200_0.5", "second_3000",
                "second_1500"]


def assert_second_chance_ran(ctx, A, B=1, b=0):
    """The peel kernel's second chance runs when the (L-1)-core of the root heuristic's best clique L has more than
    4L + 64 vertices; L comes from the device, the core is computed here."""
    h = int(ctx.clique_info(B)["heuristic_best"][b])
    assert h > 0 and _core_size(A, h - 1) > 4 * h + 64, h
    return h


@pytest.mark.parametrize("name", SEARCH_CASES)
def test_search_paths_vs_oracle(ctx, flags, name):
    A = _search_case(name)
    n = A.shape[0]
    ref = oracle(A)
    gc = check_proven(ctx, A, ref)
    if name.startswith("second"):
        assert assert_second_chance_ran(ctx, A) < len(ref)  # the root heuristic missed the planted clique
    flags(FLAG_NO_SINGLES)
    gc2, proven2, _ = single(ctx, A)
    assert proven2 == 1 and np.array_equal(gc2, gc)


def test_second_chance_clique_is_found(ctx):
    """The planted clique (1 % of the vertices, high indices, average degree) is the unique maximum."""
    rng = np.random.default_rng(31)
    A, members = second_chance_graph(2500, 0.15, 25, rng)
    gc = check_proven(ctx, A, oracle(A))
    assert np.array_equal(gc, members)
    assert assert_second_chance_ran(ctx, A) < len(members)


# ------------------------------------------------------------------ batches
def _batch_problems(n, rng):
    """About 30 problems of n vertices that take different routes: (A, reference or None, kind)."""
    probs = []
    probs.append((np.zeros((n, n), dtype=bool), np.array([], dtype=np.int32), "edgeless"))
    A = np.zeros((n, n), dtype=bool)
    A[37, n - 5] = A[n - 5, 37] = True
    probs.append((A, np.array([37, n - 5], dtype=np.int32), "edge"))
    probs.append((~np.eye(n, dtype=bool), np.arange(n, dtype=np.int32), "complete"))
    for _ in range(4):
        A, m = shortcut_graph(n, rng)
        probs.append((A, None, "shortcut"))
    for i in range(8):
        A, canon, _ = tie_graph(n, rng, word_edges=(i % 2 == 1), max_ties=SMALL_TIES)
        probs.append((A, canon, "ties"))
    for _ in range(4):
        A, _ = second_chance_graph(n, 0.15, 12, rng)
        probs.append((A, None, "second"))
    for p in (0.1, 0.2, 0.3, 0.1, 0.2, 0.05, 0.15, 0.25):
        probs.append((gnp(n, p, rng), None, "gnp"))
    for _ in range(2):
        probs.append((cocktail_party(n // 2, rng), None, "lp_closed"))
    A, _ = word_edge_graph(n, rng)
    probs.append((A, None, "word_edge"))
    for i, (A, ref, kind) in enumerate(probs):
        if ref is None and kind != "lp_closed":
            probs[i] = (A, oracle(A), kind)
    return probs


def _check_batch(ctx, probs, order):
    n = probs[0][0].shape[0]
    bits = np.stack([bits_of(probs[i][0]) for i in order])
    cl, proven, sflags = ctx.max_clique_batch(bits)
    out = {}
    for j, i in enumerate(order):
        A, ref, kind = probs[i]
        assert_clique(A, cl[j])
        if kind == "second":
            assert_second_chance_ran(ctx, A, len(order), j)
        if kind == "lp_closed":  # 2^(n/2) ties: the 50 ms first pass cannot finish, the LP bound closes it
            assert proven[j] == 2 and sflags[j] & 4, (i, proven[j], sflags[j])
            assert len(cl[j]) == n // 2
        else:
            assert proven[j] == 1, (i, kind, proven[j], sflags[j])
            assert np.array_equal(cl[j], ref), (i, kind)
        out[i] = (cl[j], proven[j])
    return out


def test_batch_mixed_routes(ctx):
    n = 256
    probs = _batch_problems(n, np.random.default_rng(77))
    B = len(probs)
    assert B >= 30
    fwd = _check_batch(ctx, probs, list(range(B)))
    rev = _check_batch(ctx, probs, list(range(B))[::-1])
    for i, (A, ref, kind) in enumerate(probs):
        if kind == "lp_closed":
            continue
        assert np.array_equal(fwd[i][0], rev[i][0])
        g1, p1, _ = single(ctx, A)  # B = 1
        assert p1 == 1 and np.array_equal(g1, fwd[i][0]), (i, kind)


def test_batch_more_problems_than_start_groups(ctx):
    """n = 4096: a bitset is 2 MB, so the L2 sizing searches 9 problems at a time (exact_conc = 9 < B = 12) and the
    persistent warps move from problem to problem with their scratch."""
    n = 4096
    rng = np.random.default_rng(4096)
    probs = []
    for i in range(12):
        if i % 2 == 0:
            A, canon, _ = tie_graph(n, rng, word_edges=(i % 4 == 0), max_ties=SMALL_TIES)
            probs.append((A, canon))
        else:
            A, _ = word_edge_graph(n, rng)
            probs.append((A, oracle(A)))
    bits = np.stack([bits_of(A) for A, _ in probs])
    cl, proven, _ = ctx.max_clique_batch(bits)
    assert ctx.clique_info(12)["exact_conc"] == 9
    cl_r, proven_r, _ = ctx.max_clique_batch(bits[::-1].copy())
    for b, (A, ref) in enumerate(probs):
        assert_clique(A, cl[b])
        assert proven[b] == 1 and np.array_equal(cl[b], ref), b
        assert proven_r[11 - b] == 1 and np.array_equal(cl_r[11 - b], ref), b
    for b in (0, 1, 11):
        g1, p1, _ = single(ctx, probs[b][0])
        assert p1 == 1 and np.array_equal(g1, cl[b])


# ------------------------------------------------------------------ the two-pass route, deterministic (flag 32768)
def _core_size(A, k):
    """Size of the k-core of A (host reference for the LP kernel's give-up rule)."""
    alive = np.ones(A.shape[0], dtype=bool)
    while True:
        deg = (A & alive[None, :]).sum(1)
        drop = alive & (deg < k)
        if not drop.any():
            return int(alive.sum())
        alive &= ~drop


def _two_pass_problems(rng):
    """Problems of 300 vertices, one per outcome of the LP kernel, plus a second re-run problem with 2^10 tied maxima
    (a complete multipartite graph of ten pairs planted in G(300, 0.2))."""
    G = gnp(300, 0.5, rng)
    cp = cocktail_party(150, rng)
    ts, omega, lp_ub = triangles_and_stars(40, [8] * 20, rng)
    assert ts.shape[0] == 300
    tied = gnp(300, 0.2, rng)
    pairs = rng.choice(300, size=20, replace=False).reshape(10, 2)
    part = np.full(300, -1)
    for j, pr in enumerate(pairs):
        part[pr] = j
    m = np.sort(pairs.ravel())
    tied[np.ix_(m, m)] = part[m][:, None] != part[m][None, :]
    return G, cp, (ts, omega, lp_ub), tied


def _check_gives_up(A, ref, c, proven, f):
    assert_clique(A, c)
    # the LP kernel gives up when 2L < |alive|: here even the (omega-1)-core is more than twice omega
    assert 2 * len(ref) < _core_size(A, len(ref) - 1)
    assert proven == 1 and f == 0, (proven, f)  # re-run canonically in the second pass: flag 2 cleared, nothing else
    assert np.array_equal(c, ref)


def _check_lp_closed(A, pairs, c, proven, f):
    assert_clique(A, c)
    assert f == 4 and proven == 2, (f, proven)
    assert len(c) == pairs


def _check_nt(A, omega, lp_ub, c, proven, f):
    assert_clique(A, c)
    # f == 0 with proven == 1 would mean the whole first pass fitted in one %globaltimer tick: flag 32768 cannot force
    # the LP route on such a problem (the graphs here need many dependent bitset reads per root)
    assert f & 8 and not f & 5 and (f >> 8) == lp_ub, (f, lp_ub)
    assert proven == 2
    assert len(c) == omega


def test_two_pass_lp_gives_up(ctx, flags):
    G, _, _, tied = _two_pass_problems(np.random.default_rng(300))
    refs = [oracle(G), oracle(tied)]
    flags(FLAG_SHORT_FIRST)
    cl, proven, f = ctx.max_clique_batch(np.stack([bits_of(G), bits_of(tied)]))
    _check_gives_up(G, refs[0], cl[0], proven[0], f[0])
    _check_gives_up(tied, refs[1], cl[1], proven[1], f[1])


@pytest.mark.parametrize("pairs", [30, 64, 150])
def test_two_pass_lp_closes(ctx, flags, pairs):
    A = cocktail_party(pairs, np.random.default_rng(pairs))
    flags(FLAG_SHORT_FIRST)
    cl, proven, f = ctx.max_clique_batch(bits_of(A)[None])
    _check_lp_closed(A, pairs, cl[0], proven[0], f[0])


@pytest.mark.parametrize("T,leaves", [(2, [20, 20]), (10, [5, 5, 5, 5]), (40, [8] * 20)])
def test_two_pass_nt_reduction(ctx, flags, T, leaves):
    assert sum(leaves) >= T + len(leaves)  # otherwise the LP kernel gives up (2L < |A|)
    A, omega, lp_ub = triangles_and_stars(T, leaves, np.random.default_rng(T))
    flags(FLAG_SHORT_FIRST)
    cl, proven, f = ctx.max_clique_batch(bits_of(A)[None])
    _check_nt(A, omega, lp_ub, cl[0], proven[0], f[0])


def test_two_pass_all_outcomes_in_one_batch(ctx, flags):
    """All outcomes in one launch sequence, in several orders: a strict (NT) problem, an LP-closed one and canonical
    re-runs share the second pass.  Whether a warp carries the strict mode into the next problem is settled by
    test_strict_mode_does_not_leak_into_the_next_problem, where only such warps reach the canonical problem."""
    G, cp, (ts, omega, lp_ub), tied = _two_pass_problems(np.random.default_rng(300))
    ref = oracle(G)
    ref_tied = oracle(tied)
    flags(FLAG_SHORT_FIRST)
    for order in ([0, 1, 2, 3], [2, 3, 0, 1], [2, 0, 1, 3], [1, 2, 3, 0, 2, 3, 2, 3]):
        mats = [(G, cp, ts, tied)[i] for i in order]
        cl, proven, f = ctx.max_clique_batch(np.stack([bits_of(A) for A in mats]))
        for j, i in enumerate(order):
            if i == 0:
                _check_gives_up(G, ref, cl[j], proven[j], f[j])
            elif i == 3:
                _check_gives_up(tied, ref_tied, cl[j], proven[j], f[j])
            elif i == 1:
                _check_lp_closed(cp, 150, cl[j], proven[j], f[j])
            else:
                _check_nt(ts, omega, lp_ub, cl[j], proven[j], f[j])


def _hidden_tie_problem(n, rng, k=10):
    """Sparse G(n, 0.01) with two tied k-cliques: X at high indices, its members given ~150 extra edges so that the root
    heuristic (top-degree roots) finds it; Y at lower indices with ordinary degrees.  The canonical answer is Y, the
    heuristic incumbent is X: only the exact search turns one into the other."""
    A = gnp(n, 0.01, rng)
    X = np.sort(rng.choice(np.arange(n - n // 16, n), size=k, replace=False))
    Y = np.sort(rng.choice(np.arange(n // 8, n // 2), size=k, replace=False))
    for v in X:
        others = rng.choice(n // 2, size=150, replace=False)
        A[v, others] = A[others, v] = True
    plant(A, X)
    plant(A, Y)
    return A, X, Y


def test_strict_mode_does_not_leak_into_the_next_problem(ctx, flags):
    """Second pass, n = 4096, B = 12: 9 start groups, so problem 3 has none and is reached only by warps that swept
    through the strict (NT) problem 2 before it.  Problem 3 is a canonical re-run whose heuristic incumbent is a
    non-canonical tie.  A warp that kept problem 2's strict mode would take problem 3's roots under a stop bound of 0
    and search none of them, leaving the incumbent in place."""
    n, B = 4096, 12
    rng = np.random.default_rng(12)
    ts, omega, _ = triangles_and_stars(2, [2044, 2044], rng)
    H, X, Y = _hidden_tie_problem(n, rng)
    ref = oracle(H)
    assert np.array_equal(ref, Y) and Y[0] < X[0]
    empty = np.zeros((n, n), dtype=bool)
    mats = [empty, empty, ts, H] + [empty] * (B - 4)
    bits = np.stack([bits_of(A) for A in mats])
    heur, _ = ctx.max_clique(bits[3], n, mode=1)  # the heuristic incumbent alone
    assert np.array_equal(heur, X)
    flags(FLAG_SHORT_FIRST)
    cl, proven, f = ctx.max_clique_batch(bits)
    conc = ctx.clique_info(B)["exact_conc"]
    assert conc == 9 and 3 not in {k * B // conc for k in range(conc)}
    assert f[2] & 8 and proven[2] == 2 and len(cl[2]) == omega, (f[2], proven[2])
    assert proven[3] == 1 and f[3] == 0, (proven[3], f[3])
    assert_clique(H, cl[3])
    assert np.array_equal(cl[3], ref)
    for b in [0, 1] + list(range(4, B)):
        assert len(cl[b]) == 0 and proven[b] == 1


# ------------------------------------------------------------------ depth cap (flag 65536)
def test_depth_cap_is_reported(ctx, flags):
    A = cocktail_party(12, np.random.default_rng(12))  # about 12 levels deep
    flags(FLAG_DEPTH8)
    cl, proven, f = ctx.max_clique_batch(bits_of(A)[None])
    assert_clique(A, cl[0])
    assert len(cl[0]) <= 12
    assert proven[0] != 1
    # the depth-cap bit; or, if the 50 ms first pass ran out first, the LP bound closed the problem
    assert (f[0] & 1) or (f[0] & 4 and proven[0] == 2), f[0]


def test_depth_cap_leaves_shallow_searches_alone(ctx, flags):
    rng = np.random.default_rng(8)
    cases = [shortcut_graph(300, rng)[0], gnp(150, 0.1, rng)]
    refs = [oracle(A) for A in cases]
    plain = [single(ctx, A) for A in cases]
    flags(FLAG_DEPTH8)
    for A, ref, (g0, p0, _) in zip(cases, refs, plain):
        g, p, f = single(ctx, A)
        assert p == p0 == 1 and f == 0
        assert np.array_equal(g, g0) and np.array_equal(g, ref)


# ------------------------------------------------------------------ input contract
def _dirty(bits, n):
    """Set every bit at or beyond n in each row's last word, and every diagonal bit."""
    d = bits.copy()
    if n % 64:
        d[..., -1] |= np.uint64(~((1 << (n % 64)) - 1) & ((1 << 64) - 1))
    idx = np.arange(n)
    d[..., idx, idx // 64] |= (np.uint64(1) << (idx % 64).astype(np.uint64))
    return d


@pytest.mark.parametrize("n", [33, 100, 128, 1000])
def test_stray_and_diagonal_bits_are_ignored(ctx, n):
    rng = np.random.default_rng(500 + n)
    mats = [word_edge_graph(n, rng)[0], tie_graph(n, rng)[0], shortcut_graph(n, rng, k=min(12, n // 3))[0]]
    clean = np.stack([bits_of(A) for A in mats])
    dirty = _dirty(clean, n)
    assert not np.array_equal(clean, dirty)
    cl0, p0, f0 = ctx.max_clique_batch(clean)
    cl1, p1, f1 = ctx.max_clique_batch(dirty)
    for b, A in enumerate(mats):
        assert_clique(A, cl1[b])
        assert np.array_equal(cl0[b], cl1[b]) and p0[b] == p1[b] == 1
        assert np.array_equal(cl0[b], oracle(A))
        g, p = ctx.max_clique(dirty[b], n)
        assert p and np.array_equal(g, cl0[b])


# ------------------------------------------------------------------ whole path: two tied motions
def _two_motion_scene(seed, k=20, n_out=40, nb=0.01):
    """Two disjoint groups of k correspondences under two different rigid motions, plus outliers: two tied maximum
    cliques.  Returns (src, dst, expected clique = the group with the lower minimum index, its motion)."""
    rng = np.random.default_rng(seed)
    n = 2 * k + n_out
    src = rng.uniform(-1, 1, size=(n, 3))
    perm = rng.permutation(n)
    ga, gb, out = np.sort(perm[:k]), np.sort(perm[k:2 * k]), perm[2 * k:]
    dst = np.empty_like(src)
    motions = []
    for g in (ga, gb):
        R, t = synth.random_rotation(rng), rng.uniform(-2, 2, size=3)
        e = rng.normal(size=(k, 3))
        e *= (0.5 * nb * rng.uniform(size=(k, 1)) ** (1 / 3)) / np.linalg.norm(e, axis=1, keepdims=True)
        dst[g] = src[g] @ R.T + t + e
        motions.append((R, t))
    dst[out] = rng.uniform(-3, 3, size=(n_out, 3))
    first = 0 if ga[0] < gb[0] else 1
    return src, dst, (ga, gb)[first], motions[first], nb


def _params(mod, nb):
    return mod.default_params(noise_bound=nb, cbar2=1.0, estimate_scaling=0, rotation_estimation_algorithm=0,
                              rotation_gnc_factor=1.4, rotation_max_iterations=100, rotation_cost_threshold=1e-12)


def _check_scene(o, clique, proven, R, t, expect, motion):
    assert np.array_equal(clique, expect)
    assert np.array_equal(clique, o["clique"])
    assert proven == 1
    assert synth.angular_error(o["R"], R) <= ROT_TOL
    assert np.linalg.norm(o["t"] - t) <= TRANS_TOL
    assert synth.angular_error(motion[0], R) < 0.05 and np.linalg.norm(motion[1] - t) < 0.05


def test_solve_two_tied_motions(ctx):
    src, dst, expect, motion, nb = _two_motion_scene(0)
    o = orc.solve(src, dst, _params(orc, nb))
    g = ctx.solve(src, dst, _params(capi, nb))
    assert g["valid"]
    _check_scene(o, g["clique"], g["sol"].clique_proven_optimal, g["R"], g["t"], expect, motion)


@pytest.mark.parametrize("B", [8, 64])
def test_solve_batch_two_tied_motions(ctx, B):
    scenes = [_two_motion_scene(100 * B + b) for b in range(B)]
    nb = scenes[0][4]
    src = np.ascontiguousarray(np.stack([s[0] for s in scenes]))
    dst = np.ascontiguousarray(np.stack([s[1] for s in scenes]))
    sols, cl = ctx.solve_batch_array(src, dst, _params(capi, nb))
    for b, (s, d, expect, motion, _) in enumerate(scenes):
        o = orc.solve(s, d, _params(orc, nb))
        m = int(sols[b]["clique_size"])
        _check_scene(o, cl[b, :m], int(sols[b]["clique_proven_optimal"]), capi.rotation_from_solution_record(sols[b]),
                     np.asarray(sols[b]["translation"]), expect, motion)
