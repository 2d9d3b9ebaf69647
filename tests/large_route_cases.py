"""Graphs for the large clique route, with their exact cores and what the device's capped peels leave (plain numpy).

A case is an undirected edge list on n vertices; `to_bits` packs it into the (n, words64(n)) uint64 rows that
`tzr_max_clique(_batch)` takes, without any n x n array, so the builders work at n = 65536.  The references here work
on the edge list: the exact k-core by layered peeling to convergence, core numbers, and two lower bounds on the
survivors of a peel stopped after r rounds:
- layered rounds (`peel_to_core` in the small route's peel kernel): every vertex of the set is tested against the
  degrees at the start of the round, so a pendant path loses exactly one vertex per round from its free end;
- in-place rounds (`core_round_kernel` on the large route): a warp scans a word's vertices in ascending order, four at
  a time, and removals are visible at once.  On a path numbered in descending index order from its free end, a vertex
  goes only after its higher neighbour, which the same warp scans later, so at most one vertex goes per round, or two
  when a warp working on the next word removes the end first.  The bound allows two per round for every path.
Both peels start from {v : deg v >= k}, which removes each path's free end before the first round.
"""
import numpy as np

U64 = np.uint64


def words64(n):
    return (n + 63) // 64


def _norm(edges):
    e = np.asarray(edges, dtype=np.int64).reshape(-1, 2)
    e = e[e[:, 0] != e[:, 1]]
    e = np.sort(e, axis=1)
    return np.unique(e, axis=0) if len(e) else e


def clique_edges(members):
    m = np.asarray(members, dtype=np.int64)
    i, j = np.triu_indices(len(m), 1)
    return np.stack([m[i], m[j]], axis=1)


def to_bits(n, edges):
    bits = np.zeros((n, words64(n)), dtype=U64)
    e = _norm(edges)
    for a, b in ((e[:, 0], e[:, 1]), (e[:, 1], e[:, 0])):
        np.bitwise_or.at(bits, (a, b >> 6), U64(1) << (b & 63).astype(U64))
    return bits


def edges_of_bits(bits, n):
    """Edge list (i < j) of a bitset, by row chunks (the inverse of to_bits; used to check it)."""
    out = []
    for r0 in range(0, n, 1024):
        rows = np.unpackbits(bits[r0:r0 + 1024].view(np.uint8), axis=1, bitorder="little")[:, :n]
        i, j = np.nonzero(rows)
        keep = r0 + i < j
        out.append(np.stack([r0 + i[keep], j[keep]], axis=1))
    return np.concatenate(out) if out else np.zeros((0, 2), dtype=np.int64)


def degrees(n, edges):
    e = _norm(edges)
    return np.bincount(e.ravel(), minlength=n)


def _alive_degrees(n, e, alive):
    both = alive[e[:, 0]] & alive[e[:, 1]]
    return np.bincount(e[both].ravel(), minlength=n)


def layered_peel(n, edges, k, rounds=None):
    """Layered peeling of {deg >= k} (the start counts as round 0), stopped after `rounds` more rounds (None: to
    convergence).  Returns (sorted survivors, rounds that removed something after the start)."""
    e = _norm(edges)
    alive = degrees(n, e) >= k
    r = 0
    while rounds is None or r < rounds:
        drop = alive & (_alive_degrees(n, e, alive) < k)
        if not drop.any():
            break
        alive &= ~drop
        r += 1
    return np.nonzero(alive)[0], r


def kcore(n, edges, k):
    return layered_peel(n, edges, k)[0]


def core_numbers(n, edges):
    """Core number of every vertex (largest k whose k-core holds it), by peeling the k-cores in turn."""
    e = _norm(edges)
    core = np.zeros(n, dtype=np.int64)
    alive = np.ones(n, dtype=bool)
    k = 0
    while alive.any():
        k += 1
        while True:
            drop = alive & (_alive_degrees(n, e, alive) < k)
            if not drop.any():
                break
            alive &= ~drop
        core[alive] = k
    return core


def innermost_core(n, edges):
    c = core_numbers(n, edges)
    return np.nonzero(c == c.max())[0]


def layered_survivors_bound(core_size, path_lengths, rounds):
    """Survivors of `rounds` layered rounds after the start on a core with pendant paths of these lengths."""
    return core_size + sum(max(0, p - 1 - rounds) for p in path_lengths)


def inplace_survivors_bound(core_size, path_lengths, rounds):
    """Fewest survivors of `rounds` in-place rounds after the start, under the most favourable warp interleaving."""
    return core_size + sum(max(0, p - 1 - 2 * rounds) for p in path_lengths)


# ------------------------------------------------------------------ builders
def pendant_paths(n, clique, paths):
    """Clique `clique` with pendant paths.  paths: list of (first, length); path p holds first ... first + length - 1,
    hangs from clique[p % len(clique)] at `first` and ends at first + length - 1: numbered in descending index order
    from its free end.  The (|clique| - 1)-core is the clique (for |clique| = 3: the 2-core of a triangle with trees)."""
    clique = np.sort(np.asarray(clique, dtype=np.int64))
    parts = [clique_edges(clique)]
    used = set(clique.tolist())
    lengths = []
    for p, (first, length) in enumerate(paths):
        v = np.arange(first, first + length, dtype=np.int64)
        assert v[-1] < n and not used & set(v.tolist()), (first, length)
        used |= set(v.tolist())
        parts.append(np.array([[clique[p % len(clique)], first]]))
        parts.append(np.stack([v[:-1], v[1:]], axis=1))
        lengths.append(length)
    L = len(clique)
    return dict(n=n, edges=_norm(np.concatenate(parts)), clique=clique, L=L, core=clique, paths=lengths)


def filler_case(n, clique, filler, offsets, attach, remainder=(), rng=None):
    """A clique K_L (vertices `clique`) next to a filler on the vertices `filler` (N of them, N even): the circulant
    graph on filler positions with the given odd offsets (each < N / 2), bipartite between even and odd positions, so
    triangle-free and 2 |offsets|-regular.  Clique member i is joined to `attach` filler vertices of its own, all at even
    positions (pairwise non-adjacent), which lifts its degree above the filler's: the greedy's top-degree root lies in
    the clique.  `remainder` vertices are paired off into single edges (degree 1, below L - 1), in a random order.
    With 2 |offsets| >= L - 1 and L >= 3:
    - the (L - 1)-core is clique | filler, exactly;
    - the clique is the unique maximum clique: a clique with two filler vertices has one at an odd position, which no
      clique member sees, and a filler vertex sees one clique member at most;
    - the second chance of the peel kernel drops the plain filler vertices in its first round (their degree is below
      the mean), the attached ones in its second, and ends on the clique (`second_chance_rounds`)."""
    clique = np.sort(np.asarray(clique, dtype=np.int64))
    filler = np.asarray(filler, dtype=np.int64)
    L, N = len(clique), len(filler)
    offsets = [int(s) for s in offsets]
    assert N % 2 == 0 and all(s % 2 == 1 and s < N // 2 for s in offsets) and len(set(offsets)) == len(offsets)
    assert 2 * len(offsets) >= L - 1 and L - 1 + attach > 2 * len(offsets) + 1 and L * attach <= N // 2
    pos = np.arange(N)
    parts = [clique_edges(clique)]
    parts += [np.stack([filler[pos], filler[(pos + s) % N]], axis=1) for s in offsets]
    ev = filler[0::2]
    parts.append(np.stack([np.repeat(clique, attach), ev[:L * attach]], axis=1))
    rem = np.asarray(remainder, dtype=np.int64)
    if len(rem) >= 2:
        rem = (rng or np.random.default_rng(0)).permutation(rem)
        parts.append(rem[:len(rem) // 2 * 2].reshape(-1, 2))
    core = np.sort(np.concatenate([clique, filler]))
    return dict(n=n, edges=_norm(np.concatenate(parts)), clique=clique, L=L, core=core, paths=[],
                filler_degree=2 * len(offsets), attach=attach)


def odd_offsets(N, count, rng):
    return sorted(int(s) for s in rng.choice(np.arange(1, N // 2, 2), size=count, replace=False))


def core_of_size(n, size, L, rng, special=(), clique_ranks=None, pool=None):
    """filler_case whose (L - 1)-core has exactly `size` vertices (size - L even), placed at random indices of `pool`
    (default [0, n)) that include `special`; clique_ranks: positions of the clique members among the sorted core
    (default: random)."""
    d = L - 1 + (L - 1) % 2                      # the filler's degree: the least even number >= L - 1
    attach = d + 3 - L
    special = np.asarray(sorted(set(special)), dtype=np.int64)
    pool = np.arange(n) if pool is None else np.asarray(pool)
    others = rng.choice(np.setdiff1d(pool, special), size=size - len(special), replace=False)
    core = np.sort(np.concatenate([special, others]))
    ranks = np.asarray(clique_ranks if clique_ranks is not None else rng.choice(size, size=L, replace=False))
    assert len(ranks) == L
    clique = core[np.sort(ranks)]
    filler = rng.permutation(np.setdiff1d(core, clique))
    case = filler_case(n, clique, filler, odd_offsets(size - L, d // 2, rng), attach,
                       np.setdiff1d(np.arange(n), core), rng)
    assert np.array_equal(case["core"], core)
    return case


def second_chance_rounds(n, edges, alive, L, max_rounds=64):
    """The peel kernel's second chance on the set `alive`: drop every vertex below the mean in-set degree while the
    mean is below 3/4 of |S| - 1, else the minimum-degree vertices (or the lowest vertex when nothing goes), until S is
    a clique or |S| <= L.  Returns (rounds, final set)."""
    e = _norm(edges)
    S = np.zeros(n, dtype=bool)
    S[alive] = True
    for r in range(max_rounds):
        cnt = int(S.sum())
        if cnt <= L:
            return r, np.nonzero(S)[0]
        d = _alive_degrees(n, e, S)[S]
        tot, dmin = int(d.sum()), int(d.min())
        if dmin == cnt - 1:
            return r, np.nonzero(S)[0]
        idx = np.nonzero(S)[0]
        drop = (d * cnt < tot) if tot * 4 < 3 * cnt * (cnt - 1) else (d == dmin)
        if not drop.any():
            drop = np.arange(cnt) == 0
        S[idx[drop]] = False
    return max_rounds, np.nonzero(S)[0]


# ------------------------------------------------------------------ the cases the GPU tests run
WORD_EDGES = np.array([32 * k + r for k in range(2048) for r in (0, 31)])


def slow_peel_case(name):
    """Pendant paths on a triangle (clique number 3, 2-core = the triangle)."""
    if name == "one300":     # the small route's 256 layered rounds leave 43 path vertices, 48 in-place rounds >= 203
        return pendant_paths(400, [0, 31, 399], [(32, 300)])
    if name == "lp260":      # the capped layered peel leaves 6 vertices: the LP kernel's bound is within reach
        return pendant_paths(300, [0, 1, 2], [(3, 260)])
    if name == "several":    # 64 ... 600 vertices, starting and ending at word edges
        return pendant_paths(4096, [31, 32, 4095], [(64, 64), (128, 97), (256, 255), (1024, 300), (2047, 600),
                                                    (3001, 451), (3500, 500)])
    if name == "paths250":   # n = 65536: 250 paths of 256 on the triangle {0, 31, 65535}
        return pendant_paths(65536, [0, 31, 65535], [(32 + 256 * p, 256) for p in range(250)])
    raise KeyError(name)


def cap_case(size, n):
    """An (L - 1)-core of exactly `size` vertices: L = 5 or 6 below 1000 vertices, 9 or 10 above (size - L even)."""
    L = (5 if size < 1000 else 9) + (size % 2 == 0)
    return core_of_size(n, size, L, np.random.default_rng(size + n))


def word_edge_case(n):
    """Clique members at compacted positions 31, 32, 63, 64, 1023, 1024 and the last one (vertex n - 1); at n = 65536
    every core member lies at v % 32 in {0, 31}, at n = 4096 the core holds the word edges 0, 31, 32, 63, 1023, 1024,
    2047, 2048 and n - 1."""
    K = 1537
    ranks = [31, 32, 63, 64, 1023, 1024, K - 1]
    if n == 65536:
        return core_of_size(n, K, 7, np.random.default_rng(7), special=(0, 31, 32767, 32768, 65535),
                            clique_ranks=ranks, pool=WORD_EDGES)
    return core_of_size(n, K, 7, np.random.default_rng(8), special=(0, 31, 32, 63, 1023, 1024, 2047, 2048, n - 1),
                        clique_ranks=ranks)


def mixed_batch_cases(n=36000):
    """One batch of n-vertex problems that leave the large route every way: (name, case, expected route)."""
    rng = np.random.default_rng(36)
    edgeless = dict(n=n, edges=np.zeros((0, 2), dtype=np.int64), clique=np.zeros(0, dtype=np.int64), L=0,
                    core=np.zeros(0, dtype=np.int64), paths=[])
    shortcut = pendant_paths(n, [5, 64, 900, 901, 2047, 2048, 30000, n - 1], [(100, 40), (3000, 90), (n - 60, 50)])
    slow = pendant_paths(n, [33, 34, 35], [(1000, 300), (5000, 600)])
    return [("edgeless", edgeless, 1), ("shortcut", shortcut, 8), ("core200", core_of_size(n, 200, 6, rng), 200),
            ("slow", slow, 3), ("core1200", core_of_size(n, 1200, 8, rng), 1200),
            ("above_cap", core_of_size(n, 32769, 9, rng), -1)]


# ------------------------------------------------------------------ a two-motion registration scene
def two_motion_scene(n, m, seed, nb=0.01):
    """n correspondences: two disjoint groups of m under two rigid motions (noise below nb / 2), the rest with targets
    spread over a 100 m cube, where two of them rarely keep a source distance.  The exact inlier graph (edge iff
    | |s_i - s_j| - |d_i - d_j| | <= 2 nb) comes from the pairs whose targets lie within the largest source distance
    plus 2 nb of each other (no other pair can be an edge); `margin` is the smallest distance of any such pair's
    residual from the threshold."""
    from scipy.spatial import cKDTree
    rng = np.random.default_rng(seed)
    src = rng.uniform(-1, 1, size=(n, 3))
    dst = rng.uniform(-50, 50, size=(n, 3))
    perm = rng.permutation(n)
    groups = [np.sort(perm[:m]), np.sort(perm[m:2 * m])]
    motions = []
    for g in groups:
        q = rng.normal(size=4)
        q /= np.linalg.norm(q)
        w, x, y, z = q
        R = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                      [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                      [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])
        t = rng.uniform(-2, 2, size=3)
        e = rng.normal(size=(m, 3))
        e *= 0.5 * nb * rng.uniform(size=(m, 1)) / np.linalg.norm(e, axis=1, keepdims=True)
        dst[g] = src[g] @ R.T + t + e
        motions.append((R, t))
    pairs = np.array(sorted(cKDTree(dst).query_pairs(2 * np.sqrt(3) + 2 * nb + 1e-9)), dtype=np.int64).reshape(-1, 2)
    res = np.abs(np.linalg.norm(src[pairs[:, 0]] - src[pairs[:, 1]], axis=1)
                 - np.linalg.norm(dst[pairs[:, 0]] - dst[pairs[:, 1]], axis=1))
    edges = pairs[res <= 2 * nb]
    margin = float(np.min(np.abs(res - 2 * nb))) if len(res) else np.inf
    first = 0 if groups[0][0] < groups[1][0] else 1
    return dict(n=n, src=src, dst=dst, nb=nb, groups=groups, motions=motions, edges=_norm(edges), margin=margin,
                expect=groups[first], motion=motions[first], m=m)
