"""CPU-side checks of certifying the last solve: tzr_last_inliers and tzr_certify_last_solve are exported with the
argument order the binding uses (the ABI version stays 2), and the argument checks that need no device reject."""
import ctypes as C
import importlib
import os
import re

import numpy as np
import pytest

capi = importlib.import_module("teaser-plusplus_b200.capi")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _ensure_built():
    if not os.path.exists(capi.LIB_PATH):
        capi.build()


def _header_args(name):
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "teaser_b200.h")).read(), flags=re.S)
    m = re.search(r"int\s+" + name + r"\s*\(([^)]*)\)", hdr)
    assert m, f"{name} missing from the header"
    return [a.split()[-1].lstrip("*") for a in " ".join(m.group(1).split()).split(",")]


def test_symbols_exported():
    _ensure_built()
    L = C.CDLL(capi.LIB_PATH)
    for name in ("tzr_last_inliers", "tzr_certify_last_solve"):
        assert hasattr(L, name) and name in capi._SYMBOLS
    assert capi.lib().tzr_abi_version() == 2


def test_argtypes_follow_the_header():
    _ensure_built()
    L = capi.lib()
    dp, u8p, i32p, i64p = C.POINTER(C.c_double), C.POINTER(C.c_uint8), C.POINTER(C.c_int32), C.POINTER(C.c_int64)
    assert _header_args("tzr_last_inliers") == ["ctx", "b", "rot_inliers", "trans_inliers", "n_rot", "n_trans"]
    assert L.tzr_last_inliers.argtypes == [C.c_void_p, C.c_int, u8p, u8p, i64p, i32p]
    assert _header_args("tzr_certify_last_solve") == ["ctx", "params", "count", "problems", "results", "status",
                                                      "traj", "traj_capacity"]
    assert L.tzr_certify_last_solve.argtypes == [C.c_void_p, C.POINTER(capi.CertifierParams), C.c_int, i32p,
                                                 C.POINTER(capi.CertificationResult), i32p, C.POINTER(dp), i32p]


def test_rejected_without_a_device():
    _ensure_built()
    L = capi.lib()
    p = capi.CertifierParams()
    L.tzr_certifier_params_default(C.byref(p))
    res = (capi.CertificationResult * 2)()
    probs = np.array([0, 1], dtype=np.int32)
    n_rot, n_trans = C.c_int64(7), C.c_int32(7)
    # no context
    assert L.tzr_last_inliers(None, 0, None, None, C.byref(n_rot), C.byref(n_trans)) == capi.TZR_ERR_INVALID_ARG
    assert n_rot.value == 7 and n_trans.value == 7  # nothing written
    assert L.tzr_certify_last_solve(None, C.byref(p), 2, capi._p(probs, C.c_int32), res, None, None,
                                    None) == capi.TZR_ERR_INVALID_ARG
    # trajectories without capacities, or no results: rejected before the context is looked at
    traj = (C.POINTER(C.c_double) * 2)()
    assert L.tzr_certify_last_solve(None, C.byref(p), 2, None, res, None, traj, None) == capi.TZR_ERR_INVALID_ARG
    assert L.tzr_certify_last_solve(None, C.byref(p), 2, None, None, None, None, None) == capi.TZR_ERR_INVALID_ARG


@pytest.mark.parametrize("bad", [[], [[0, 1]], [0.5, 1.0], "ab"])
def test_problem_lists_validated(bad):
    with pytest.raises(capi.TzrError):
        capi.Context._certify_last_problems(bad)


def test_problem_list_normalised():
    assert capi.Context._certify_last_problems(None) is None
    pr = capi.Context._certify_last_problems((3, 0, 3))
    assert pr.dtype == np.int32 and pr.flags.c_contiguous and pr.tolist() == [3, 0, 3]
