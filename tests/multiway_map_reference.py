"""The host form of the fused map's first step (DESIGN.md §3.25): every cloud of a sequence transformed by its pose,
each coordinate float32(((R_r0 x + R_r1 y) + R_r2 z) + t_r) in float64 with x, y, z read exactly, the clouds
concatenated in order.  The library downsamples this concatenation exactly as tzr_voxel_downsample(_colors)_batch."""
import numpy as np


def transform_concat(clouds, poses):
    """(sum n, 3) float32: cloud k by the (4,4) float64 pose poses[k], in the library's operation order."""
    out = []
    for cloud, T in zip(clouds, poses):
        p = np.asarray(cloud, dtype=np.float32).astype(np.float64)
        T = np.asarray(T, dtype=np.float64)
        cols = [((T[r, 0] * p[:, 0] + T[r, 1] * p[:, 1]) + T[r, 2] * p[:, 2]) + T[r, 3] for r in range(3)]
        out.append(np.stack(cols, axis=1).astype(np.float32))
    return np.concatenate(out) if out else np.zeros((0, 3), dtype=np.float32)
