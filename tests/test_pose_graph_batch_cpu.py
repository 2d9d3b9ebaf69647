"""CPU checks of the batched GNC-TLS pose graph (tzr_pose_graph_optimize_batch): exported, declared with its argument
names and bound in capi; a call without a context refused; the binding's own argument checks.  The entry's call-level
refusals need a context and are checked in test_gpu_pose_graph_batch.py."""
import ctypes as C
import importlib
import os
import re

import numpy as np
import pytest

capi = importlib.import_module("teaser-plusplus_b200.capi")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAME = "tzr_pose_graph_optimize_batch"
ARGS = ["ctx", "params", "G", "K", "E", "edges", "edge_transforms", "information", "uncertain", "initial_poses",
        "poses", "weights", "inlier_mask", "residuals", "summaries", "status"]


@pytest.fixture(scope="module")
def header():
    if not os.path.exists(capi.LIB_PATH):
        capi.build()
    return open(os.path.join(ROOT, "include", "teaser_b200.h")).read()


def test_symbol_exported_declared_and_bound(header):
    code = re.sub(r"/\*.*?\*/", "", header, flags=re.S)
    m = re.search(r"int\s+%s\s*\(([^)]*)\)" % NAME, code)
    assert m, f"{NAME} missing from the header"
    args = [a.split()[-1].lstrip("*") for a in " ".join(m.group(1).split()).split(",")]
    assert args == ARGS
    assert NAME in capi._SYMBOLS
    assert len(getattr(capi.lib(), NAME).argtypes) == len(ARGS)
    assert callable(capi.Context.optimize_pose_graph_batch)


def one_graph():
    """The arrays of one two-node graph, and status (initialised to 7)"""
    i32 = C.POINTER(C.c_int32)
    keep = dict(K=np.array([2], dtype=np.int32), E=np.array([1], dtype=np.int32),
                ed=np.array([[0, 1]], dtype=np.int32), tr=(capi.Similarity * 1)(capi.similarity(None)),
                info=np.eye(6).ravel(), poses=(capi.Similarity * 2)(), status=np.full(1, 7, dtype=np.int32))
    ptrs = dict(K=keep["K"].ctypes.data_as(i32), E=keep["E"].ctypes.data_as(i32),
                edges=(i32 * 1)(keep["ed"].ctypes.data_as(i32)),
                transforms=(C.POINTER(capi.Similarity) * 1)(C.cast(keep["tr"], C.POINTER(capi.Similarity))),
                information=(C.POINTER(C.c_double) * 1)(keep["info"].ctypes.data_as(C.POINTER(C.c_double))),
                poses=(C.POINTER(capi.Similarity) * 1)(C.cast(keep["poses"], C.POINTER(capi.Similarity))),
                status=keep["status"].ctypes.data_as(i32))
    return keep, ptrs


def call(ctx, prm, G=1, **null):
    """The entry on one_graph() with the arrays named in null passed as NULL; returns (rc, status[0], whether any pose
    was written).  test_gpu_pose_graph_batch.py calls it with a context."""
    keep, p = one_graph()
    for k in null:
        p[k] = None
    rc = getattr(capi.lib(), NAME)(ctx, C.byref(prm), G, p["K"], p["E"], p["edges"], p["transforms"],
                                   p["information"], None, None, p["poses"], None, None, None, None, p["status"])
    return rc, int(keep["status"][0]), any(bytes(keep["poses"]))


def test_null_context_refused():
    assert call(None, capi.pose_graph_params(0.05)) == (capi.TZR_ERR_INVALID_ARG, 7, False)  # nothing written


def _deviceless_context():
    ctx = object.__new__(capi.Context)
    ctx._h = C.c_void_p()
    return ctx


@pytest.mark.parametrize("case", ["transforms", "uncertain"])
def test_python_checks_need_no_device(case):
    """Raised by the binding before the entry is called (its message, not the library's)"""
    g = dict(K=3, edges=[(0, 1), (1, 2)], transforms=[np.eye(4)] * 2, information=[np.eye(6)] * 2)
    if case == "transforms":
        g["transforms"] = [np.eye(4)]
    else:
        g["uncertain"] = [0, 1, 1]
    with pytest.raises(capi.TzrError, match="per edge"):
        _deviceless_context().optimize_pose_graph_batch([g], 0.05)
