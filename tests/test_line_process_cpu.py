"""CPU checks of the line-process C-ABI (tzr_pose_graph_optimize_line_process,
tzr_register_cloud_pairs_multiway_line_process): exported, declared with the argument lists the Python binding passes
and listed among the symbols capi.lib() checks; the structs' layouts and Open3D's defaults; the stop-reason codes; calls
without a context refused."""
import ctypes as C
import importlib
import os
import re

import numpy as np
import pytest

import line_process_reference as lp

capi = importlib.import_module("teaser-plusplus_b200.capi")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

CHAIN = ["ctx", "fparams", "params", "n_clouds", "n", "pts", "P", "pair_clouds", "tuple_seeds", "solutions", "status",
         "problem_index", "n_corr", "corr", "cliques", "global_scale", "icp", "colors", "lambda_geometric", "kernel",
         "icp_results"]
ARGS = {
    "tzr_pose_graph_optimize_line_process": ["ctx", "params", "K", "E", "edges", "edge_transforms", "information",
                                             "uncertain", "initial_poses", "poses", "confidence", "kept", "residuals",
                                             "summary"],
    "tzr_register_cloud_pairs_multiway_line_process": CHAIN + ["uncertain", "lp", "information", "info_counts",
                                                               "edge_confidence", "edge_kept", "poses", "lp_summary",
                                                               "lp_status"],
}


@pytest.fixture(scope="module")
def header():
    if not os.path.exists(capi.LIB_PATH):
        capi.build()
    return open(os.path.join(ROOT, "include", "teaser_b200.h")).read()


@pytest.mark.parametrize("name", sorted(ARGS))
def test_symbol_exported_declared_and_bound(header, name):
    code = re.sub(r"/\*.*?\*/", "", header, flags=re.S)
    m = re.search(r"int\s+%s\s*\(([^)]*)\)" % name, code)
    assert m, f"{name} missing from the header"
    args = [a.split()[-1].lstrip("*") for a in " ".join(m.group(1).split()).split(",")]
    assert args == ARGS[name]
    assert name in capi._SYMBOLS
    assert len(getattr(capi.lib(), name).argtypes) == len(ARGS[name])


def test_struct_layouts_defaults_and_stop_codes(header):
    assert C.sizeof(capi.LineProcessParams) == 88 and C.sizeof(capi.LineProcessSummary) == 56
    for f, _ in capi.LineProcessParams._fields_:
        assert f in header
    p = capi.line_process_params(0.05)
    assert p.max_correspondence_distance == 0.05
    for k, v in lp.DEFAULTS.items():
        assert getattr(p, k) == v, k
    raw = capi.LineProcessParams()
    capi.lib().tzr_line_process_params_default(C.byref(raw))
    assert raw.max_correspondence_distance == 0
    capi.lib().tzr_line_process_params_default(None)
    for name, code in lp.STOP.items():
        assert capi.LP_STOP[code] == name
        assert re.search(r"#define TZR_LP_STOP_\w+ %d\b" % code, header)


def test_null_context_refused():
    L = capi.lib()
    prm = capi.line_process_params(0.05)
    ed = np.array([[0, 1]], dtype=np.int32)
    tr = capi.similarity(None)
    info = np.eye(6).ravel()
    poses = (capi.Similarity * 2)()
    assert L.tzr_pose_graph_optimize_line_process(None, C.byref(prm), 2, 1, ed.ctypes.data_as(C.POINTER(C.c_int32)),
                                                  C.byref(tr), info.ctypes.data_as(C.POINTER(C.c_double)), None, None,
                                                  poses, None, None, None, None) == capi.TZR_ERR_INVALID_ARG
    args = [None] * len(L.tzr_register_cloud_pairs_multiway_line_process.argtypes)
    assert len(args) == 30
    args[3] = args[6] = 1
    args[18] = 0.0
    assert L.tzr_register_cloud_pairs_multiway_line_process(*args) == capi.TZR_ERR_INVALID_ARG
