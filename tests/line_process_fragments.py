"""Pose graphs shaped like the fragments of Open3D's reconstruction system (make_fragments): odometry between
consecutive frames and loop closures between keyframes, built on line_process_graphs.graph."""
import numpy as np

from line_process_graphs import graph


def fragment(seed, K, n_wrong=0, noise=0.003, points=(100, 400)):
    """A graph shaped like one fragment of Open3D's make_fragments: odometry (k, k + 1), loop closures between each
    keyframe (every 5th node) and the next two keyframes, then n_wrong wrong closures between keyframes more than 10
    nodes apart, last.  Returns graph()'s tuple."""
    keys = list(range(0, K, 5))
    extra = [(a, b) for a in keys for b in keys if a < b <= a + 10]
    far = [(a, b) for a in keys for b in keys if b > a + 10]
    rng = np.random.default_rng(seed + 7919)
    wrong = [far[i] for i in sorted(rng.choice(len(far), size=n_wrong, replace=False))] if n_wrong else []
    return graph(seed, K, extra, wrong=wrong, noise=noise, points=points)
