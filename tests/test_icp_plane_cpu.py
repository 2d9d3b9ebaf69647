"""CPU checks of the point-to-plane ICP and normals C-ABI (tzr_estimate_normals(_batch), tzr_icp_point_to_plane(_batch),
tzr_register_cloud_pairs_icp_point_to_plane): the entry points are exported, declared in the header with the argument
lists the Python binding passes and listed among the symbols capi.lib() checks; malformed calls are refused before any
device work."""
import ctypes as C
import importlib
import os
import re

import numpy as np
import pytest

capi = importlib.import_module("teaser-plusplus_b200.capi")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

ARGS = {
    "tzr_estimate_normals": ["ctx", "pts", "n", "normal_search_radius", "normals_out"],
    "tzr_estimate_normals_batch": ["ctx", "B", "n", "pts", "normal_search_radius", "normals_out", "status"],
    "tzr_icp_point_to_plane": ["ctx", "params", "src", "ns", "dst", "nd", "dst_normals", "init", "result", "corr"],
    "tzr_icp_point_to_plane_batch": ["ctx", "params", "B", "ns", "src", "nd", "dst", "dst_normals", "init", "results",
                                     "corr"],
    "tzr_register_cloud_pairs_icp_point_to_plane": ["ctx", "fparams", "params", "n_clouds", "n", "pts", "P",
                                                    "pair_clouds", "tuple_seeds", "solutions", "status",
                                                    "problem_index", "n_corr", "corr", "cliques", "global_scale",
                                                    "icp", "icp_results"],
}

fp, i32p = C.POINTER(C.c_float), C.POINTER(C.c_int32)


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


def test_chained_entry_takes_the_point_to_point_arguments(header):
    m = re.search(r"int\s+tzr_register_cloud_pairs_icp\s*\(([^)]*)\)", header)
    q = re.search(r"int\s+tzr_register_cloud_pairs_icp_point_to_plane\s*\(([^)]*)\)", header)
    assert " ".join(m.group(1).split()) == " ".join(q.group(1).split())


def _icp_batch(ctx, p, B=2, ns=4, nd=4, normals="ok"):
    x = np.zeros((max(ns, 1), 3), dtype=np.float32)
    y = np.zeros((max(nd, 1), 3), dtype=np.float32)
    nrm = np.zeros((max(nd, 1), 4), dtype=np.float32)
    Bn = max(B, 1)
    n_s = np.full(Bn, ns, dtype=np.int32)
    n_d = np.full(Bn, nd, dtype=np.int32)
    init = (capi.Similarity * Bn)(*[capi.similarity(None) for _ in range(Bn)])
    res = (capi.IcpResult * Bn)()
    xs = (fp * Bn)(*[x.ctypes.data_as(fp)] * Bn)
    ys = (fp * Bn)(*[y.ctypes.data_as(fp)] * Bn)
    if normals == "null":
        ns_ = None
    else:
        ns_ = (fp * Bn)(*[nrm.ctypes.data_as(fp)] * Bn)
        if normals == "null_entry":
            ns_[Bn - 1] = None
    return capi.lib().tzr_icp_point_to_plane_batch(ctx, C.byref(p), B, n_s.ctypes.data_as(i32p), xs,
                                                   n_d.ctypes.data_as(i32p), ys, ns_, init, res, None)


@pytest.mark.parametrize("case", ["null_ctx", "null_normals", "null_normals_entry", "r_zero", "r_negative", "r_nan",
                                  "iter_negative", "B_zero", "ns_zero", "nd_zero"])
def test_icp_argument_checks_need_no_device(case):
    """Malformed calls return TZR_ERR_INVALID_ARG without a device (the context is NULL here, and every argument check
    runs before the device is touched)."""
    p = capi.icp_params(0.1)
    kw = {}
    if case == "null_normals":
        kw["normals"] = "null"
    elif case == "null_normals_entry":
        kw["normals"] = "null_entry"
    elif case == "r_zero":
        p.max_correspondence_distance = 0.0
    elif case == "r_negative":
        p.max_correspondence_distance = -1.0
    elif case == "r_nan":
        p.max_correspondence_distance = float("nan")
    elif case == "iter_negative":
        p.max_iteration = -1
    elif case == "B_zero":
        kw["B"] = 0
    elif case == "ns_zero":
        kw["ns"] = 0
    elif case == "nd_zero":
        kw["nd"] = 0
    assert _icp_batch(None, p, **kw) == capi.TZR_ERR_INVALID_ARG
    x = np.zeros((3, 3), dtype=np.float32)
    nrm = np.zeros((3, 4), dtype=np.float32)
    res = capi.IcpResult()
    single_normals = None if case == "null_normals" else nrm.ctypes.data_as(fp)
    assert capi.lib().tzr_icp_point_to_plane(None, C.byref(p), x.ctypes.data_as(fp), 3, x.ctypes.data_as(fp), 3,
                                             single_normals, None, C.byref(res), None) == capi.TZR_ERR_INVALID_ARG


@pytest.mark.parametrize("case", ["null_ctx", "radius_zero", "radius_negative", "radius_nan", "B_zero", "n_zero",
                                  "null_out", "null_out_entry"])
def test_normals_argument_checks_need_no_device(case):
    x = np.zeros((4, 3), dtype=np.float32)
    out = np.zeros((4, 4), dtype=np.float32)
    r, B, n = 0.1, 2, np.array([4, 4], dtype=np.int32)
    outs = (fp * 2)(out.ctypes.data_as(fp), out.ctypes.data_as(fp))
    if case == "radius_zero":
        r = 0.0
    elif case == "radius_negative":
        r = -1.0
    elif case == "radius_nan":
        r = float("nan")
    elif case == "B_zero":
        B = 0
    elif case == "n_zero":
        n[1] = 0
    elif case == "null_out":
        outs = None
    elif case == "null_out_entry":
        outs[1] = None
    pts = (fp * 2)(x.ctypes.data_as(fp), x.ctypes.data_as(fp))
    L = capi.lib()
    assert L.tzr_estimate_normals_batch(None, B, n.ctypes.data_as(i32p), pts, r, outs, None) == capi.TZR_ERR_INVALID_ARG
    single_out = None if case in ("null_out", "null_out_entry") else out.ctypes.data_as(fp)
    single_n = 0 if case == "n_zero" else 4
    assert L.tzr_estimate_normals(None, x.ctypes.data_as(fp), single_n, r, single_out) == capi.TZR_ERR_INVALID_ARG


def test_chained_entry_refuses_null_icp_params():
    L = capi.lib()
    assert L.tzr_register_cloud_pairs_icp_point_to_plane(None, None, None, 0, None, None, 0, None, None, None, None,
                                                         None, None, None, None, None, None, None) == \
        capi.TZR_ERR_INVALID_ARG


def test_python_normals_shapes():
    """(nd,3) normals get a zero curvature column; other shapes are refused before the library is called."""
    n3 = np.arange(12, dtype=np.float32).reshape(4, 3)
    n4 = capi._normals32(n3, 4, "t")
    assert n4.shape == (4, 4) and np.array_equal(n4[:, :3], n3) and not n4[:, 3].any()
    with pytest.raises(capi.TzrError):
        capi._normals32(np.zeros((4, 5), dtype=np.float32), 4, "t")
    with pytest.raises(capi.TzrError):
        capi._normals32(np.zeros((3, 4), dtype=np.float32), 4, "t")
