"""numpy restatement of the voxel-grid downsampling that tzr_voxel_downsample(_batch) computes (include/teaser_b200.h,
DESIGN.md §3.12), bit-exact by construction.

Per cloud, all arithmetic is IEEE float64 with no FMA contraction:
- Inputs: n float xyz points, read exactly as float64, and one voxel_size v (finite, > 0).
- Finite points only: a point with any non-finite coordinate belongs to no voxel (trace -1) and does not affect the
  bounds.
- Bounds: min and max are the component-wise bounds over the finite points; vmin = min - (v * 0.5),
  vmax = max + (v * 0.5).
- Too small a voxel: v * INT_MAX < max_k (vmax_k - vmin_k) is TZR_ERR_TOO_LARGE (Open3D's check).
- Voxel index: i_k = (int) floor((p_k - vmin_k) / v), a division.
- Grid-size limit: points are grouped by the exact triple (i_x, i_y, i_z); a cloud whose per-axis voxel counts
  (i_k of its largest finite coordinate, + 1) multiply to more than 2^62 is TZR_ERR_TOO_LARGE.
- Output point: the sum of the voxel's members, added one at a time in ascending input index starting from 0.0,
  divided by (double) count, rounded once to float.
- Output order: voxels ordered by their first (lowest-index) member.

The sum runs rank by rank, vectorised over voxels: iteration k adds every voxel's k-th member (members sorted by
(voxel, index)), so each voxel's sum runs in index order, exactly as the one-at-a-time loop.
"""
import numpy as np

INT_MAX = 2147483647
CELL_LIMIT = 1 << 62
TZR_OK = 0
TZR_ERR_TOO_LARGE = -6


def voxel_indices(p64, vmin, v):
    """(int) floor((p - vmin) / v) per coordinate: the division, as Open3D writes it."""
    return np.floor((p64 - vmin) / v).astype(np.int64)


def grid(pts, v):
    """(status, vmin, counts, finite mask) of one cloud: the bounds, the INT_MAX check and the 2^62-cell limit."""
    p = np.asarray(pts, dtype=np.float32).astype(np.float64)
    fin = np.isfinite(p).all(axis=1)
    if not fin.any():
        return TZR_OK, None, None, fin
    lo = p[fin].min(axis=0)
    hi = p[fin].max(axis=0)
    h = v * 0.5
    vmin = lo - h
    vmax = hi + h
    if v * INT_MAX < (vmax - vmin).max():
        return TZR_ERR_TOO_LARGE, vmin, None, fin
    counts = [int(c) + 1 for c in voxel_indices(hi, vmin, v)]
    if counts[0] * counts[1] * counts[2] > CELL_LIMIT:
        return TZR_ERR_TOO_LARGE, vmin, counts, fin
    return TZR_OK, vmin, counts, fin


def downsample(pts, v):
    """(points (m,3) float32, trace (n,) int32, status) of one cloud."""
    p32 = np.ascontiguousarray(pts, dtype=np.float32).reshape(-1, 3)
    n = p32.shape[0]
    trace = np.full(n, -1, dtype=np.int32)
    status, vmin, counts, fin = grid(p32, v)
    if status != TZR_OK or vmin is None:
        return np.zeros((0, 3), dtype=np.float32), trace, status
    p = p32.astype(np.float64)
    members = np.flatnonzero(fin)
    ijk = voxel_indices(p[members], vmin, v)
    # group by the exact triple; inside a group, ascending input index
    order = np.lexsort((members, ijk[:, 2], ijk[:, 1], ijk[:, 0]))
    m_sorted = members[order]
    t_sorted = ijk[order]
    start = np.ones(len(order), dtype=bool)
    start[1:] = (t_sorted[1:] != t_sorted[:-1]).any(axis=1)
    seg = np.cumsum(start) - 1                    # voxel of every sorted member
    first = m_sorted[start]                       # lowest-index member of every voxel
    starts = np.flatnonzero(start)
    sizes = np.diff(np.append(starts, len(order)))
    row_of_voxel = np.empty(len(first), dtype=np.int64)
    row_of_voxel[np.argsort(first, kind="stable")] = np.arange(len(first))
    # rank k adds the k-th member of every voxel that has one; voxels by descending size, so those are a prefix
    by_size = np.argsort(-sizes, kind="stable")
    neg_sizes = -sizes[by_size]
    st = starts[by_size]
    acc = np.zeros((len(first), 3), dtype=np.float64)
    for k in range(int(sizes.max())):
        na = int(np.searchsorted(neg_sizes, -k, side="left"))  # voxels with more than k members
        acc[:na] = acc[:na] + p[m_sorted[st[:na] + k]]
    mean = (acc / sizes[by_size].astype(np.float64)[:, None]).astype(np.float32)
    out = np.empty_like(mean)
    out[row_of_voxel[by_size]] = mean
    trace[m_sorted] = row_of_voxel[seg].astype(np.int32)
    return out, trace, status


def downsample_dict_loop(pts, v):
    """Open3D's VoxelDownSample restated line by line with a Python dict (plus the definition's non-finite rule and
    output order): the independent check of downsample()."""
    p32 = np.ascontiguousarray(pts, dtype=np.float32).reshape(-1, 3)
    trace = [-1] * p32.shape[0]
    finite = [i for i in range(p32.shape[0]) if all(np.isfinite(float(c)) for c in p32[i])]
    if not finite:
        return np.zeros((0, 3), dtype=np.float32), np.array(trace, dtype=np.int32), TZR_OK
    lo = [min(float(p32[i][k]) for i in finite) for k in range(3)]
    hi = [max(float(p32[i][k]) for i in finite) for k in range(3)]
    vmin = [lo[k] - v * 0.5 for k in range(3)]
    vmax = [hi[k] + v * 0.5 for k in range(3)]
    if v * INT_MAX < max(vmax[k] - vmin[k] for k in range(3)):
        return np.zeros((0, 3), dtype=np.float32), np.array(trace, dtype=np.int32), TZR_ERR_TOO_LARGE
    import math
    cnt = [int(math.floor((hi[k] - vmin[k]) / v)) + 1 for k in range(3)]
    if cnt[0] * cnt[1] * cnt[2] > CELL_LIMIT:
        return np.zeros((0, 3), dtype=np.float32), np.array(trace, dtype=np.int32), TZR_ERR_TOO_LARGE
    voxels = {}      # (i, j, k) -> [sum x, sum y, sum z, count, first index]
    for i in finite:
        x = [float(c) for c in p32[i]]
        key = tuple(int(math.floor((x[k] - vmin[k]) / v)) for k in range(3))
        if key not in voxels:
            voxels[key] = [0.0, 0.0, 0.0, 0, i]
        a = voxels[key]
        a[0] += x[0]
        a[1] += x[1]
        a[2] += x[2]
        a[3] += 1
    rows = sorted(voxels.items(), key=lambda kv: kv[1][4])
    row_of = {key: r for r, (key, _) in enumerate(rows)}
    out = np.array([[a[0] / float(a[3]), a[1] / float(a[3]), a[2] / float(a[3])] for _, a in rows],
                   dtype=np.float64).astype(np.float32).reshape(-1, 3)
    for i in finite:
        x = [float(c) for c in p32[i]]
        trace[i] = row_of[tuple(int(math.floor((x[k] - vmin[k]) / v)) for k in range(3))]
    return out, np.array(trace, dtype=np.int32), TZR_OK


# ---- clouds on the definition's edges (shared by the CPU and GPU tests) ----
def lattice_on_edges(v, k=6, seed=0):
    """Points whose every coordinate lies on a voxel boundary min + (j + 1/2) v (min = 0 through the point at the
    origin), shuffled, plus the origin itself."""
    rng = np.random.default_rng(seed)
    j = np.stack(np.meshgrid(*[np.arange(k)] * 3, indexing="ij"), axis=-1).reshape(-1, 3)
    pts = ((j + 0.5) * v).astype(np.float32)
    pts = pts[rng.permutation(len(pts))]
    return np.concatenate([np.zeros((1, 3), np.float32), pts])


def division_case():
    """A cloud whose point x = 0.125 lies where (x - vmin) / v and (x - vmin) * (1 / v) floor to different voxels
    (v = 0.05, min = 0, so vmin = -0.025): by division it joins the point at 0.1, by the product the point at 0.16."""
    return np.array([[0.0, 0, 0], [0.1, 0, 0], [0.125, 0, 0], [0.16, 0, 0]], dtype=np.float32), 0.05
