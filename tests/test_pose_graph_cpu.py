"""CPU checks of the multiway C-ABI (tzr_information_matrix(_batch), tzr_pose_graph_optimize,
tzr_register_cloud_pairs_multiway): the entry points are exported, declared in the header with the argument lists the
Python binding passes and listed among the symbols capi.lib() checks; the structs' layouts and defaults; malformed calls
are refused before any device work."""
import ctypes as C
import importlib
import os
import re

import numpy as np
import pytest

capi = importlib.import_module("teaser-plusplus_b200.capi")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

CHAIN = ["ctx", "fparams", "params", "n_clouds", "n", "pts", "P", "pair_clouds", "tuple_seeds", "solutions", "status",
         "problem_index", "n_corr", "corr", "cliques", "global_scale", "icp", "icp_results"]
ARGS = {
    "tzr_information_matrix": ["ctx", "src", "ns", "dst", "nd", "transform", "max_correspondence_distance",
                               "information", "count"],
    "tzr_information_matrix_batch": ["ctx", "B", "ns", "src", "nd", "dst", "transforms",
                                     "max_correspondence_distance", "information", "counts"],
    "tzr_pose_graph_optimize": ["ctx", "params", "K", "E", "edges", "edge_transforms", "information", "uncertain",
                                "initial_poses", "poses", "weights", "inlier_mask", "residuals", "summary"],
    "tzr_register_cloud_pairs_multiway": CHAIN + ["uncertain", "pg", "information", "info_counts", "edge_weights",
                                                  "edge_mask", "poses", "pg_summary", "pg_status"],
}


@pytest.fixture(scope="module")
def header():
    if not os.path.exists(capi.LIB_PATH):
        capi.build()
    return re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "teaser_b200.h")).read(), flags=re.S)


@pytest.mark.parametrize("name", sorted(ARGS))
def test_symbol_exported_declared_and_bound(header, name):
    m = re.search(r"int\s+%s\s*\(([^)]*)\)" % name, header)
    assert m, f"{name} missing from the header"
    args = [a.split()[-1].lstrip("*") for a in " ".join(m.group(1).split()).split(",")]
    assert args == ARGS[name]
    assert name in capi._SYMBOLS
    assert len(getattr(capi.lib(), name).argtypes) == len(ARGS[name])
    assert "#define TZR_ABI_VERSION 2" in header


def test_struct_layouts_and_defaults(header):
    assert C.sizeof(capi.PoseGraphParams) == 40 and C.sizeof(capi.PoseGraphSummary) == 16
    for f in ("max_correspondence_distance", "gnc_factor", "cost_threshold", "max_iterations",
              "max_inner_iterations", "reference_node"):
        assert f in header
    p = capi.pose_graph_params(0.05)
    assert (p.max_correspondence_distance, p.gnc_factor, p.cost_threshold) == (0.05, 1.4, 1e-6)
    assert (p.max_iterations, p.max_inner_iterations, p.reference_node) == (100, 10, 0)
    raw = capi.PoseGraphParams()
    capi.lib().tzr_pose_graph_params_default(C.byref(raw))
    assert raw.max_correspondence_distance == 0  # no default distance
    capi.lib().tzr_pose_graph_params_default(None)  # tolerated


def test_null_context_refused():
    L = capi.lib()
    x = np.zeros((4, 3), dtype=np.float32)
    fp = C.POINTER(C.c_float)
    info = np.zeros(36)
    cnt = C.c_int32(0)
    tr = capi.similarity(None)
    assert L.tzr_information_matrix(None, x.ctypes.data_as(fp), 4, x.ctypes.data_as(fp), 4, C.byref(tr), 0.1,
                                    info.ctypes.data_as(C.POINTER(C.c_double)), C.byref(cnt)) == capi.TZR_ERR_INVALID_ARG
    ns = np.array([4], dtype=np.int32)
    assert L.tzr_information_matrix_batch(None, 1, ns.ctypes.data_as(C.POINTER(C.c_int32)), (fp * 1)(x.ctypes.data_as(fp)),
                                          ns.ctypes.data_as(C.POINTER(C.c_int32)), (fp * 1)(x.ctypes.data_as(fp)),
                                          C.byref(tr), 0.1, info.ctypes.data_as(C.POINTER(C.c_double)),
                                          None) == capi.TZR_ERR_INVALID_ARG
    pg = capi.pose_graph_params(0.05)
    ed = np.array([[0, 1]], dtype=np.int32)
    poses = (capi.Similarity * 2)()
    assert L.tzr_pose_graph_optimize(None, C.byref(pg), 2, 1, ed.ctypes.data_as(C.POINTER(C.c_int32)), C.byref(tr),
                                     info.ctypes.data_as(C.POINTER(C.c_double)), None, None, poses, None, None, None,
                                     None) == capi.TZR_ERR_INVALID_ARG
    args = [None] * len(L.tzr_register_cloud_pairs_multiway.argtypes)
    assert len(args) == 27
    args[3] = args[6] = 1  # n_clouds, P
    assert L.tzr_register_cloud_pairs_multiway(*args) == capi.TZR_ERR_INVALID_ARG
    # the checks that need a context (the multiway entry's own arguments, the pose graph's ranges and messages) run on
    # the device: tests/test_gpu_pose_graph.py::test_argument_checks_with_a_context
