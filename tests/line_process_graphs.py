"""Synthetic pose graphs for the line-process tests: ground-truth poses, noisy odometry and loop closures in the
cloud-pair orientation (p_d ~ T_sd p_s), information matrices from random overlap points, and Open3D's tutorial rule
for uncertainty (pair (k, k + 1) certain, every other pair uncertain)."""
import numpy as np
from scipy.spatial.transform import Rotation

import pose_graph_reference as pg


def rigid(rng, angle=0.3, shift=0.5):
    T = np.eye(4)
    T[:3, :3] = Rotation.from_rotvec(rng.normal(size=3) * angle).as_matrix()
    T[:3, 3] = rng.normal(size=3) * shift
    return T


def graph(seed, K, extra, wrong=(), noise=0.002, complete=False, points=(100, 400)):
    """(gt, edges (E,2) int32, T (E,4,4), L (E,6,6), uncertain): a chain 0-1-...-(K-1) plus extra pairs (or every pair
    when complete), then the wrong closures, whose T_sd is off by a large random motion."""
    rng = np.random.default_rng(seed)
    gt = [np.eye(4)] + [rigid(rng) for _ in range(K - 1)]
    pairs = [(a, b) for a in range(K) for b in range(K) if a < b] if complete else \
        [(k, k + 1) for k in range(K - 1)] + list(extra)
    edges, T, L, unc = [], [], [], []
    for s, d in list(pairs) + list(wrong):
        Tsd = pg.inv(gt[d]) @ gt[s]
        Tsd = (rigid(rng, 0.5, 1.0) if (s, d) in wrong else rigid(rng, noise, noise)) @ Tsd
        pts = rng.uniform(-1, 1, size=(int(rng.integers(*points)), 3))
        S = np.einsum("ni,nj->ij", pts, pts)
        m = pts.sum(axis=0)
        Lam = np.zeros((6, 6))  # sum over the points of G^T G, G = [-[q]x | I]
        Lam[:3, :3] = np.trace(S) * np.eye(3) - S
        Lam[:3, 3:] = -pg.skew(m).T
        Lam[3:, :3] = -pg.skew(m)
        Lam[3:, 3:] = len(pts) * np.eye(3)
        edges.append((s, d))
        T.append(Tsd)
        L.append(Lam)
        unc.append(0 if d == s + 1 else 1)
    return gt, np.array(edges, dtype=np.int32), T, L, unc
