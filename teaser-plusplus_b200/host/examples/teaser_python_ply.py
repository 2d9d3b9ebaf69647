"""GPU build of the reference's Python quick-start (examples/teaser_python_ply/teaser_python_ply.py): the
`teaserpp_python` lines (Params, solver, solve, getSolution) are exactly what a TEASER++ user writes; only the PLY
reader (open3d in the reference) is replaced by this repo's 20-line ASCII parser and the RNG is seeded.

    usage: python teaser_python_ply.py <bun_zipper_res3.ply>
"""
import importlib
import os
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", "python"))
sys.path.insert(0, os.path.join(HERE, "..", "..", ".."))
import teaserpp_python  # noqa: E402

read_ply_vertices = importlib.import_module("teaser-plusplus_b200.synth").read_ply_vertices

NOISE_BOUND = 0.05
N_OUTLIERS = 1700
OUTLIER_TRANSLATION_LB = 5
OUTLIER_TRANSLATION_UB = 10


def get_angular_error(R_exp, R_est):
    return abs(np.arccos(min(max(((np.matmul(R_exp.T, R_est)).trace() - 1) / 2, -1.0), 1.0)))


if __name__ == "__main__":
    ply = sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "..", "..", "..", "tests", "golden",
                                                              "bun_zipper_res3.ply")
    rng = np.random.default_rng(1889)
    src = np.transpose(read_ply_vertices(ply).astype(np.float64))
    N = src.shape[1]
    T = np.array(
        [[9.96926560e-01, 6.68735757e-02, -4.06664421e-02, -1.15576939e-01],
         [-6.61289946e-02, 9.97617877e-01, 1.94008687e-02, -3.87705398e-02],
         [4.18675510e-02, -1.66517807e-02, 9.98977765e-01, 1.14874890e-01],
         [0, 0, 0, 1]])
    dst = T[:3, :3] @ src + T[:3, 3:4]
    dst += (rng.random((3, N)) - 0.5) * 2 * NOISE_BOUND
    outlier_indices = rng.integers(N_OUTLIERS, size=N_OUTLIERS)
    for i in range(outlier_indices.size):
        shift = OUTLIER_TRANSLATION_LB + rng.random((3, 1)) * (OUTLIER_TRANSLATION_UB - OUTLIER_TRANSLATION_LB)
        dst[:, outlier_indices[i]] += shift.squeeze()

    # ---- the reference's solver-facing code (teaser_python_ply.py:50-66)
    solver_params = teaserpp_python.RobustRegistrationSolver.Params()
    solver_params.cbar2 = 1
    solver_params.noise_bound = NOISE_BOUND
    solver_params.estimate_scaling = False
    solver_params.rotation_estimation_algorithm = \
        teaserpp_python.RobustRegistrationSolver.ROTATION_ESTIMATION_ALGORITHM.GNC_TLS
    solver_params.rotation_gnc_factor = 1.4
    solver_params.rotation_max_iterations = 100
    solver_params.rotation_cost_threshold = 1e-12
    # Not in the reference example: a safety net.  With a noise bound of 0.05 on a 0.15 m object the inlier graph of the
    # ~800 untouched points is 99 % dense; colouring-bound searches (PMC's too) do not terminate on it in reasonable
    # time (reference default limit: 3600 s).  Here the vertex-cover LP bound proves the 597-vertex clique optimal
    # right after the first 50 ms search pass, so the limit below is never reached.
    solver_params.max_clique_time_limit = 30

    solver = teaserpp_python.RobustRegistrationSolver(solver_params)
    solver.solve(src, dst)  # warm-up: CUDA context + workspace
    start = time.time()
    solver.solve(src, dst)
    end = time.time()
    solution = solver.getSolution()

    print("rotation error (rad):", get_angular_error(T[:3, :3], solution.rotation))
    print("translation error (m):", np.linalg.norm(T[:3, 3] - solution.translation))
    print("clique size:", len(solver.getInlierMaxClique()))
    print("time (s):", end - start)
