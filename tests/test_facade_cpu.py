"""CPU checks of the drop-in surfaces above the C-ABI: the pybind11 module `teaserpp_python` builds, exposes the
reference's names with the reference's defaults, and fails loudly without a GPU."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOST = os.path.join(ROOT, "teaser-plusplus_b200", "host")
sys.path.insert(0, os.path.join(HOST, "python"))


@pytest.fixture(scope="module")
def tp():
    subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "teaser-plusplus_b200", "csrc")])
    subprocess.check_call(["make", "-s", "-C", HOST])
    import teaserpp_python
    return teaserpp_python


def test_module_surface(tp):
    # names of python/teaserpp_python/teaserpp_python.cc:25-291 and __init__.py:4-58 (certifier excluded)
    for name in ("RobustRegistrationSolver", "RegistrationSolution", "RotationEstimationAlgorithm",
                 "InlierSelectionMode", "InlierGraphFormulation", "RobustRegistrationSolverParams", "OMP_MAX_THREADS"):
        assert hasattr(tp, name)
    S = tp.RobustRegistrationSolver
    assert S.ROTATION_ESTIMATION_ALGORITHM is tp.RotationEstimationAlgorithm
    assert S.INLIER_SELECTION_MODE.PMC_EXACT == tp.InlierSelectionMode.PMC_EXACT
    for meth in ("solve", "getSolution", "getInlierMaxClique", "getInlierGraph", "getRotationInliersMask",
                 "getTranslationInliersMask", "getTranslationInliers", "getRotationInliers", "getScaleInliersMask",
                 "getSrcTIMs", "getDstTIMs", "getMaxCliqueSrcTIMs", "getMaxCliqueDstTIMs", "getSrcTIMsMap",
                 "getDstTIMsMapForRotation", "getGNCRotationCostAtTermination", "getParams"):
        assert hasattr(S, meth), meth
    for prop in ("solution", "inlier_max_clique", "rotation_inliers_mask", "translation_inliers_mask", "src_tims",
                 "dst_tims", "max_clique_dst_tims", "dst_tims_map_for_rotation"):
        assert isinstance(getattr(S, prop), property) or hasattr(S, prop)


def test_params_defaults(tp):
    p = tp.RobustRegistrationSolver.Params()  # teaser/include/teaser/registration.h:419-514
    assert p.noise_bound == 0.01 and p.cbar2 == 1 and p.estimate_scaling is True
    assert p.rotation_estimation_algorithm == tp.RotationEstimationAlgorithm.GNC_TLS
    assert p.rotation_gnc_factor == 1.4 and p.rotation_max_iterations == 100 and p.rotation_cost_threshold == 1e-6
    assert p.rotation_tim_graph == tp.InlierGraphFormulation.CHAIN
    assert p.inlier_selection_mode == tp.InlierSelectionMode.PMC_EXACT
    assert p.kcore_heuristic_threshold == 0.5 and p.max_clique_time_limit == 3600
    s = tp.RobustRegistrationSolver(noise_bound=0.05, estimate_scaling=False)
    q = s.getParams()  # the reference never stores params_ (SURVEY Q1); the façade does
    assert q.noise_bound == 0.05 and q.estimate_scaling is False
    assert s.params == ()


def test_no_cpu_fallback(tp):
    try:
        import torch
        if torch.cuda.is_available():
            pytest.skip("GPU present")
    except ImportError:
        pass
    import numpy as np
    s = tp.RobustRegistrationSolver(tp.RobustRegistrationSolver.Params())
    with pytest.raises(RuntimeError):
        s.solve(np.zeros((3, 10)), np.ones((3, 10)))


@pytest.mark.parametrize("cls", ["PoseGraph", "GlobalOptimization"])
@pytest.mark.parametrize("n_init", [0, 1, 3])
def test_single_optimize_needs_one_initial_pose_per_node(tp, cls, n_init):
    # a given initial-pose list must hold num_nodes poses, an empty one included (not read as the breadth-first
    # start); refused before any device work, so with or without a GPU
    import numpy as np
    g = getattr(tp, cls)(0.05)
    with pytest.raises(ValueError, match=f"teaser::{cls}::optimize: one initial pose per node"):
        g.optimize(2, [(0, 1)], [np.eye(4)], [np.eye(6)], initial_poses=[np.eye(4)] * n_init)


def test_mex_shim_compiles_against_stub():
    """matlab/teaser_mex.cc (MATLAB absent here): syntax/type check against a stub of the MEX API."""
    mex = os.path.join(HOST, "matlab")
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    subprocess.check_call([cxx, "-std=c++17", "-fsyntax-only", "-DTZR_MEX_SYNTAX_CHECK", "-I", mex,
                           "-I", os.path.join(ROOT, "include"), os.path.join(mex, "teaser_mex.cc")])


def test_ply_io_roundtrip(tmp_path):
    """teaser::PLYReader / PLYWriter of the façade (reference: test/teaser/io-test.cc) — host-only code, runs here."""
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    exe = str(tmp_path / "ply_io_test")
    subprocess.check_call([cxx, "-std=c++17", "-O1", "-I", os.path.join(HOST, "include"),
                           os.path.join(ROOT, "tests", "cpp", "ply_io_test.cc"), os.path.join(HOST, "src", "ply_io.cc"),
                           "-o", exe])
    golden = os.path.join(ROOT, "tests", "golden")
    out = subprocess.run([exe, os.path.join(golden, "cube.ply"), os.path.join(golden, "bun_zipper_res3.ply"),
                          str(tmp_path)], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0 and out.stdout.strip() == "ok", out.stdout + out.stderr
