"""Independent numpy restatement of Matcher::calculateCorrespondences (reference teaser/src/matcher.cc:55-297), for
the correspondence stage's boundary tests (csrc/matcher.cu; DESIGN.md 3.8).

Written from the reference's control flow, not from oracle/matcher_oracle.cc or the kernels:

* normalizePoints (:55-113): the mean is one float32 addition chain per coordinate in index order (np.add.accumulate
  is strictly sequential, unlike np.add.reduce, which sums pairwise), divided by float(n).  Norms are
  (x*x + y*y) + z*z in float32.  `temp > max_scale` lets neither NaN nor 0 win; global_scale_ is 1 with
  use_absolute_scale, and the points are divided by it whenever it is not 1 (also when it is 0, NaN or inf).
* Nearest neighbours: flann::L2<float> order, groups of four ((d0^2 + d1^2) + d2^2) + d3^2 added to the running sum,
  then the tail.  The lowest index wins among equal distances and a NaN distance never beats a number.
* advancedMatching (:114-297): the larger cloud is "i" (strictly: nd > ns swaps); i_to_j for the hit i only;
  corres = corres_ij ++ corres_ji; the cross check as the Mi/Mj triple loop; the tuple test over 100 * ncorr trials
  with corres_tuple pushes; swap back, sort, unique.
* The tuple test's draws: the project replaces srand(time(NULL)); rand() % ncorr by the top 31 bits of
  splitmix64(seed + 3 t + k), k = 0..2, in uint64 arithmetic that wraps (documented in the oracle's header)."""
import numpy as np

F32 = np.float32
U64 = np.uint64
M64 = (1 << 64) - 1


# ---- normalizePoints -----------------------------------------------------------------------------------------------
def sequential_mean(p):
    """mean = mean + p over the points in index order, then mean / npti (float32)."""
    p = np.asarray(p, dtype=F32).reshape(-1, 3)
    with np.errstate(all="ignore"):
        s = np.add.accumulate(p, axis=0, dtype=F32)[-1]
        return (s / F32(p.shape[0])).astype(F32)


def norms(p):
    """Vector3f::norm() of every row: sqrt((x*x + y*y) + z*z) in float32."""
    p = np.asarray(p, dtype=F32)
    with np.errstate(all="ignore"):
        x, y, z = p[:, 0], p[:, 1], p[:, 2]
        return np.sqrt((x * x + y * y) + z * z).astype(F32)


def max_scale(p, mean):
    """max over the cloud of ||p - mean|| under `temp > max_scale` from 0: NaN never wins."""
    with np.errstate(all="ignore"):
        t = norms(np.asarray(p, dtype=F32) - mean)
    t = t[~np.isnan(t)]
    m = t.max() if t.size else F32(0)
    return F32(m) if m > 0 else F32(0)


def global_scale(src, dst, use_absolute_scale=False, mean=sequential_mean):
    """Matcher::global_scale_.  `mean` replaces the sequential mean (tests use it to show that a different
    summation order would change the scale's bits)."""
    if use_absolute_scale:
        return F32(1.0)
    scale = F32(0)
    for p in (src, dst):
        m = max_scale(p, np.asarray(mean(p), dtype=F32))
        if m > scale:
            scale = m
    return scale


def normalize_points(src, dst, use_absolute_scale):
    """The centred and rescaled clouds and global_scale_."""
    out = []
    for p in (src, dst):
        p = np.asarray(p, dtype=F32)
        with np.errstate(all="ignore"):
            out.append((p - sequential_mean(p)).astype(F32))
    g = global_scale(src, dst, use_absolute_scale)
    if g != F32(1.0):
        with np.errstate(all="ignore"):
            out = [(p / g).astype(F32) for p in out]
    return out[0], out[1], g


# ---- nearest neighbours ----------------------------------------------------------------------------------------------
def l2_flann(q, db):
    """(m, n) float32 distances in flann::L2<float>'s order."""
    q = np.asarray(q, dtype=F32)
    db = np.asarray(db, dtype=F32)
    dim = q.shape[1]
    res = np.zeros((q.shape[0], db.shape[0]), dtype=F32)
    with np.errstate(all="ignore"):
        k = 0
        while k + 3 < dim:
            d = [q[:, None, k + u] - db[None, :, k + u] for u in range(4)]
            res = res + (((d[0] * d[0] + d[1] * d[1]) + d[2] * d[2]) + d[3] * d[3])
            k += 4
        for k in range(k, dim):
            d = q[:, None, k] - db[None, :, k]
            res = res + d * d
    return res


def nn1(q, db, chunk_elems=1 << 22):
    """Index of the nearest db row of every q row: lowest index among equal distances, NaN never beats a number
    (an all-NaN row gives 0)."""
    q = np.asarray(q, dtype=F32)
    out = np.zeros(q.shape[0], dtype=np.int64)
    step = max(1, chunk_elems // max(1, db.shape[0]))
    for a in range(0, q.shape[0], step):
        d = l2_flann(q[a:a + step], db)
        nan = np.isnan(d)
        dn = np.where(nan, F32(np.inf), d)
        idx = np.argmin(dn, axis=1)
        rows = np.arange(d.shape[0])
        inf_rows = np.isinf(dn[rows, idx])
        for r in np.nonzero(inf_rows)[0]:          # an inf distance still beats NaN; all NaN keeps index 0
            cand = np.nonzero(~nan[r])[0]
            idx[r] = cand[0] if cand.size else 0
        out[a:a + step] = idx
    return out


def tie_count(q, db):
    """How many q rows have more than one db row at their minimal distance."""
    n = 0
    for a in range(0, q.shape[0], 256):
        d = l2_flann(q[a:a + 256], db)
        n += int(((d == np.nanmin(d, axis=1, keepdims=True)).sum(1) > 1).sum())
    return n


# ---- advancedMatching ------------------------------------------------------------------------------------------------
def correspondences(ns, nd, src_feat, dst_feat, use_crosscheck):
    """(swapped, corres (k, 2) in (i, j) indices and the reference's list order, hit i mask) of :114-216."""
    swapped = nd > ns
    fi, fj = (dst_feat, src_feat) if swapped else (src_feat, dst_feat)
    n_i, n_j = (nd, ns) if swapped else (ns, nd)
    nn_of_j = nn1(fj, fi)                                   # searchKDTree(&feature_tree_i, features_[fj][j])
    i_to_j = np.full(n_i, -1, dtype=np.int64)
    hit = np.zeros(n_i, dtype=bool)
    hit[nn_of_j] = True
    hi = np.nonzero(hit)[0]
    if hi.size:
        i_to_j[hi] = nn1(fi[hi], fj)                        # only for the i some j chose (:155-159)
    corres_ij = [(i, int(i_to_j[i])) for i in range(n_i) if i_to_j[i] != -1]
    corres_ji = [(int(nn_of_j[j]), j) for j in range(n_j)]
    corres = corres_ij + corres_ji
    if use_crosscheck:
        Mi = [[] for _ in range(n_i)]
        Mj = [[] for _ in range(n_j)]
        for ci, cj in corres_ij:
            Mi[ci].append(cj)
        for ci, cj in corres_ji:
            Mj[cj].append(ci)
        corres = []
        for i in range(n_i):
            for j in Mi[i]:
                for c in Mj[j]:
                    if c == i:
                        corres.append((i, j))
    return swapped, np.array(corres, dtype=np.int64).reshape(-1, 2), hit


def splitmix64(x):
    """splitmix64 of a uint64 array, wrapping."""
    x = np.asarray(x, dtype=U64) + U64(0x9E3779B97F4A7C15)
    x = (x ^ (x >> U64(30))) * U64(0xBF58476D1CE4E5B9)
    x = (x ^ (x >> U64(27))) * U64(0x94D049BB133111EB)
    return x ^ (x >> U64(31))


def draws(seed, ncorr):
    """(100 * ncorr, 3) indices into corres: (splitmix64(seed + 3 t + k) >> 33) % ncorr."""
    t = np.arange(100 * ncorr, dtype=U64)
    base = U64(int(seed) & M64) + U64(3) * t                 # uint64 wrap-around, as in C
    r = np.stack([splitmix64(base + U64(k)) >> U64(33) for k in range(3)], axis=1)
    return (r % U64(max(ncorr, 1))).astype(np.int64)


def dist3(a, b):
    with np.errstate(all="ignore"):
        d = (a - b).astype(F32)
        return np.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]).astype(F32)


def tuple_trials(src, dst, src_feat, dst_feat, use_absolute_scale, use_crosscheck, tuple_scale, seed):
    """Every trial of the tuple test: dict(corres (i, j), r (trials, 3), li, lj (trials, 3), passed (trials,),
    swapped, g).  The trial list exists whenever the test runs (use_tuple_test and tuple_scale != 0)."""
    ps, pd, g = normalize_points(src, dst, use_absolute_scale)
    swapped, corres, hit = correspondences(len(ps), len(pd), src_feat, dst_feat, use_crosscheck)
    pi, pj = (pd, ps) if swapped else (ps, pd)
    ncorr = len(corres)
    r = draws(seed, ncorr)
    s = F32(tuple_scale)
    li = np.zeros((len(r), 3), dtype=F32)
    lj = np.zeros((len(r), 3), dtype=F32)
    if ncorr:
        ci, cj = corres[:, 0], corres[:, 1]
        for e, (u, v) in enumerate(((0, 1), (1, 2), (2, 0))):
            li[:, e] = dist3(pi[ci[r[:, u]]], pi[ci[r[:, v]]])
            lj[:, e] = dist3(pj[cj[r[:, u]]], pj[cj[r[:, v]]])
    with np.errstate(all="ignore"):
        passed = np.all((li * s < lj) & (lj < li / s), axis=1)
    return dict(corres=corres, r=r, li=li, lj=lj, passed=passed, swapped=swapped, g=g, hit=hit)


def match(src, dst, src_feat, dst_feat, use_absolute_scale=True, use_crosscheck=True, use_tuple_test=True,
          tuple_scale=0.0, tuple_seed=0):
    """(pairs (m, 2) int32 in (source, target) order, sorted and unique; global_scale_ as np.float32)."""
    src = np.asarray(src, dtype=F32)
    dst = np.asarray(dst, dtype=F32)
    if use_tuple_test and F32(tuple_scale) != 0:
        tr = tuple_trials(src, dst, src_feat, dst_feat, use_absolute_scale, use_crosscheck, tuple_scale, tuple_seed)
        corres, swapped, g = tr["corres"], tr["swapped"], tr["g"]
        kept = tr["r"][tr["passed"]].reshape(-1)               # corres_tuple: the three entries of every pass
        corres = corres[kept] if len(kept) else np.zeros((0, 2), dtype=np.int64)
    else:
        g = normalize_points(src, dst, use_absolute_scale)[2]
        swapped, corres, _ = correspondences(len(src), len(dst), src_feat, dst_feat, use_crosscheck)
    if swapped:
        corres = corres[:, ::-1]
    pairs = np.unique(corres.reshape(-1, 2), axis=0) if len(corres) else np.zeros((0, 2), dtype=np.int64)
    return pairs.astype(np.int32), F32(g)


# ---- other summation orders (premises: a kernel that summed this way would change the scale's bits) ------------------
def pairwise_mean(p):
    """float32 mean by recursive halving (a tree reduction)."""
    p = np.asarray(p, dtype=F32).reshape(-1, 3)

    def tree(a):
        if a.shape[0] == 1:
            return a[0]
        h = a.shape[0] // 2
        return (tree(a[:h]) + tree(a[h:])).astype(F32)

    with np.errstate(all="ignore"):
        return (tree(p) / F32(p.shape[0])).astype(F32)


def float64_mean(p):
    return np.asarray(p, dtype=np.float64).reshape(-1, 3).mean(0).astype(F32)


def lane_strided_mean(p):
    """32 lane partial sums (lane l adds the points l, l + 32, ...) combined by an xor butterfly, lane 0's value."""
    p = np.asarray(p, dtype=F32).reshape(-1, 3)
    s = np.zeros((32, 3), dtype=F32)
    with np.errstate(all="ignore"):
        for i in range(p.shape[0]):
            s[i % 32] = s[i % 32] + p[i]
        off = 16
        while off:
            s = (s + s[np.arange(32) ^ off]).astype(F32)
            off >>= 1
        return (s[0] / F32(p.shape[0])).astype(F32)


# ---- cases -----------------------------------------------------------------------------------------------------------
def offset_clouds(n, seed, n_dst=40, dim=4):
    """A source of n points at 1e4 + unit-scale spread with one point 50 away, and a 40-point target of half that
    spread: the global scale is the far point's distance from a mean whose float32 ulp is 2^-10, so it follows the
    mean's last bits.  dim-4 descriptors keep the nearest-neighbour reference cheap at large n."""
    rng = np.random.default_rng(seed)
    src = (1.0e4 + rng.uniform(-1, 1, size=(n, 3))).astype(F32)
    src[n // 2] = (1.0e4 + np.array([50.0, -30.0, 20.0]) + rng.uniform(-1, 1, size=3)).astype(F32)
    dst = (1.0e4 + rng.uniform(-0.5, 0.5, size=(n_dst, 3))).astype(F32)
    sf = rng.normal(size=(n, dim)).astype(F32)
    tf = rng.normal(size=(n_dst, dim)).astype(F32)
    return src, dst, sf, tf


def triangle_pair(lj, li=10.0, y=4.0):
    """Three correspondences, exactly centred (the sums are exact, so the mean is 0) and with use_absolute_scale not
    rescaled.  Source ("i") A = (-li, y, 0), B = (0, y, 0), C = (li, -2y, 0); target the same with lj.  |AB| is
    sqrt(fl(l^2)) = l exactly; |BC| and |CA| are the other two sides.  Descriptor k is the same on both sides and far
    from the other two, so the correspondences are (0, 0), (1, 1), (2, 2)."""
    def cloud(l):
        l = F32(l)
        return np.array([[-l, y, 0], [0, y, 0], [l, -2 * y, 0]], dtype=F32)

    feat = (np.eye(3, 33) * 100).astype(F32)
    return cloud(li), cloud(lj), feat, feat.copy()


def last_pair_case(ns, nd, seed):
    """A matcher problem whose last source and last target share a descriptor no other point is near, so that
    (ns - 1, nd - 1) is a mutual nearest-neighbour pair."""
    import importlib
    synth = importlib.import_module("teaser-plusplus_b200.synth")
    mp = synth.matcher_problem(ns, nd, min(ns, nd) // 3, seed=seed)
    sf, tf = mp["src_feat"].copy(), mp["dst_feat"].copy()
    sf[-1] = tf[-1] = F32(300.0)
    return mp["src_pts"], mp["dst_pts"], sf, tf


def hub_case(ns=500, nd=300, hub=123, seed=3):
    """Every target's nearest source descriptor is source `hub`: the other sources sit 1000 away."""
    import importlib
    synth = importlib.import_module("teaser-plusplus_b200.synth")
    mp = synth.matcher_problem(ns, nd, 0, seed=seed)
    sf = (mp["src_feat"] + F32(1000)).astype(F32)
    sf[hub] = mp["dst_feat"].mean(0)
    return mp["src_pts"], mp["dst_pts"], sf, mp["dst_feat"]


def duplicate_case(seed=5, n0=700):
    """Every descriptor several times on both sides, the copies hundreds of rows apart (different nearest-neighbour
    segments): the lowest index among equal distances decides every nearest neighbour and so which pairs are
    mutual."""
    import importlib
    synth = importlib.import_module("teaser-plusplus_b200.synth")
    rng = np.random.default_rng(seed)
    base = synth.random_fpfh(rng, n0, 33)
    sf = np.concatenate([base[rng.permutation(n0)], base[rng.permutation(n0)]])
    tf = np.concatenate([base[rng.permutation(n0)], base[rng.permutation(n0)[:500]]])
    mp = synth.matcher_problem(len(sf), len(tf), 200, seed=seed)
    return mp["src_pts"], mp["dst_pts"], sf, tf


def offset_seed(n):
    """The first seed whose offset clouds' global scale changes under a tree sum, a float64 mean and a lane-strided
    sum of the source (for n < 31 the first seed: so few points need not separate the orders)."""
    for seed in range(64):
        src, dst, _, _ = offset_clouds(n, seed)
        g = global_scale(src, dst).tobytes()
        if n < 31 or all(global_scale(src, dst, mean=m).tobytes() != g
                         for m in (pairwise_mean, float64_mean, lane_strided_mean)):
            return seed
    raise AssertionError(f"no offset cloud of {n} points separates the summation orders")


def nonfinite_case(kind, seed=11):
    """A 200 x 150 matcher problem with poisoned points: nan_src (one NaN coordinate in the source), nan_both (and
    one in the target), pinf / minf (one +inf target / -inf source coordinate), coincident (every point of each
    cloud the same dyadic point, so the sums are exact and every centred point is 0).  Returns the poisoned points,
    the clean points and the features."""
    import importlib
    synth = importlib.import_module("teaser-plusplus_b200.synth")
    mp = synth.matcher_problem(200, 150, 60, seed=seed)
    cs = (mp["src_pts"] * F32(3)).astype(F32)      # the clean source's scale exceeds the target's
    sp, tp = cs.copy(), mp["dst_pts"].copy()
    if kind in ("nan_src", "nan_both"):
        sp[7, 1] = np.nan
    if kind == "nan_both":
        tp[3, 0] = np.nan
    if kind == "pinf":
        tp[5, 2] = np.inf
    if kind == "minf":
        sp[0, 0] = -np.inf
    if kind == "coincident":
        sp[:] = (0.5, -2.0, 3.0)
        tp[:] = (1.25, 4.0, -0.75)
    return sp, tp, cs, mp["dst_pts"], mp["src_feat"], mp["dst_feat"]
