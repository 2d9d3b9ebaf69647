"""CPU checks of the batched line process (tzr_pose_graph_optimize_line_process_batch): exported, declared with its
argument names and bound in capi; a call without a context refused; the make_fragments-shaped graph generator."""
import ctypes as C
import importlib
import os
import re

import numpy as np
import pytest

import pose_graph_reference as pg
from line_process_fragments import fragment

capi = importlib.import_module("teaser-plusplus_b200.capi")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAME = "tzr_pose_graph_optimize_line_process_batch"
ARGS = ["ctx", "params", "G", "K", "E", "edges", "edge_transforms", "information", "uncertain", "initial_poses",
        "poses", "confidence", "kept", "residuals", "summaries", "status"]


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
    assert callable(capi.Context.global_optimization_batch)


def test_null_context_refused():
    L = capi.lib()
    prm = capi.line_process_params(0.05)
    K = np.array([2], dtype=np.int32)
    E = np.array([1], dtype=np.int32)
    ed = np.array([[0, 1]], dtype=np.int32)
    tr = (capi.Similarity * 1)(capi.similarity(None))
    info = np.eye(6).ravel()
    poses = (capi.Similarity * 2)()
    status = np.full(1, 7, dtype=np.int32)
    i32 = C.POINTER(C.c_int32)
    args = [None, C.byref(prm), 1, K.ctypes.data_as(i32), E.ctypes.data_as(i32),
            (i32 * 1)(ed.ctypes.data_as(i32)), (C.POINTER(capi.Similarity) * 1)(C.cast(tr, C.POINTER(capi.Similarity))),
            (C.POINTER(C.c_double) * 1)(info.ctypes.data_as(C.POINTER(C.c_double))), None, None,
            (C.POINTER(capi.Similarity) * 1)(C.cast(poses, C.POINTER(capi.Similarity))), None, None, None, None,
            status.ctypes.data_as(i32)]
    assert getattr(L, NAME)(*args) == capi.TZR_ERR_INVALID_ARG
    assert status[0] == 7  # nothing written


@pytest.mark.parametrize("K,n_wrong", [(100, 3), (32, 0), (128, 2), (7, 0)])
def test_fragment_generator(K, n_wrong):
    gt, edges, T, L, unc = fragment(11, K, n_wrong=n_wrong)
    pairs = [tuple(e) for e in edges.tolist()]
    keys = list(range(0, K, 5))
    closures = [(a, b) for a in keys for b in keys if a < b <= a + 10]
    assert pairs[:K - 1] == [(k, k + 1) for k in range(K - 1)]
    assert pairs[K - 1:K - 1 + len(closures)] == closures
    wrong = pairs[K - 1 + len(closures):]
    assert len(wrong) == n_wrong == len(set(wrong))
    assert all(a % 5 == 0 and b % 5 == 0 and b > a + 10 for a, b in wrong)
    assert unc == [0 if d == s + 1 else 1 for s, d in pairs]
    for j, (s, d) in enumerate(pairs):
        err = np.abs(T[j] - pg.inv(gt[d]) @ gt[s]).max()
        assert (err > 0.1) if j >= len(pairs) - n_wrong else (err < 0.05), (s, d, err)
        assert np.allclose(L[j], L[j].T) and np.all(np.linalg.eigvalsh(L[j]) > -1e-9)
    a = fragment(11, K, n_wrong=n_wrong)
    assert all(np.array_equal(x, y) for x, y in zip(a[2], T)) and np.array_equal(a[1], edges)
