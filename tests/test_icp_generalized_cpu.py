"""CPU checks of the generalized-ICP C-ABI (tzr_icp_generalized(_batch), tzr_register_cloud_pairs_icp_generalized): the
entry points are exported, declared in the header with the argument lists the Python binding passes and listed among
the symbols capi.lib() checks; malformed calls are refused before any device work."""
import ctypes as C
import importlib
import os
import re

import numpy as np
import pytest

capi = importlib.import_module("teaser-plusplus_b200.capi")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

ARGS = {
    "tzr_icp_generalized": ["ctx", "params", "epsilon", "src", "ns", "src_normals", "dst", "nd", "dst_normals", "init",
                            "result", "corr"],
    "tzr_icp_generalized_batch": ["ctx", "params", "epsilon", "B", "ns", "src", "src_normals", "nd", "dst",
                                  "dst_normals", "init", "results", "corr"],
    "tzr_register_cloud_pairs_icp_generalized": ["ctx", "fparams", "params", "n_clouds", "n", "pts", "P", "pair_clouds",
                                                 "tuple_seeds", "solutions", "status", "problem_index", "n_corr",
                                                 "corr", "cliques", "global_scale", "icp", "epsilon", "icp_results"],
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


def _icp_batch(ctx, p, epsilon=1e-3, B=2, ns=4, nd=4, src_normals="ok", dst_normals="ok"):
    x = np.zeros((max(ns, 1), 3), dtype=np.float32)
    y = np.zeros((max(nd, 1), 3), dtype=np.float32)
    sn = np.zeros((max(ns, 1), 4), dtype=np.float32)
    dn = np.zeros((max(nd, 1), 4), dtype=np.float32)
    Bn = max(B, 1)
    n_s = np.full(Bn, ns, dtype=np.int32)
    n_d = np.full(Bn, nd, dtype=np.int32)
    init = (capi.Similarity * Bn)(*[capi.similarity(None) for _ in range(Bn)])
    res = (capi.IcpResult * Bn)()
    xs = (fp * Bn)(*[x.ctypes.data_as(fp)] * Bn)
    ys = (fp * Bn)(*[y.ctypes.data_as(fp)] * Bn)

    def normals(arr, how):
        if how == "null":
            return None
        out = (fp * Bn)(*[arr.ctypes.data_as(fp)] * Bn)
        if how == "null_entry":
            out[Bn - 1] = None
        return out

    return capi.lib().tzr_icp_generalized_batch(ctx, C.byref(p), epsilon, B, n_s.ctypes.data_as(i32p), xs,
                                                normals(sn, src_normals), n_d.ctypes.data_as(i32p), ys,
                                                normals(dn, dst_normals), init, res, None)


CASES = {
    "null_ctx": {},
    "null_src_normals": dict(src_normals="null"),
    "null_src_normals_entry": dict(src_normals="null_entry"),
    "null_dst_normals": dict(dst_normals="null"),
    "null_dst_normals_entry": dict(dst_normals="null_entry"),
    "epsilon_zero": dict(epsilon=0.0),
    "epsilon_negative": dict(epsilon=-1e-3),
    "epsilon_nan": dict(epsilon=float("nan")),
    "epsilon_inf": dict(epsilon=float("inf")),
    "r_zero": {},
    "r_negative": {},
    "ns_zero": dict(ns=0),
    "nd_zero": dict(nd=0),
    "B_zero": dict(B=0),
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_icp_argument_checks_need_no_device(case):
    """Malformed calls return TZR_ERR_INVALID_ARG without a device (the context is NULL here, and every argument check
    runs before the device is touched)."""
    p = capi.icp_params(0.1)
    if case == "r_zero":
        p.max_correspondence_distance = 0.0
    elif case == "r_negative":
        p.max_correspondence_distance = -1.0
    kw = CASES[case]
    assert _icp_batch(None, p, **kw) == capi.TZR_ERR_INVALID_ARG
    ns, nd = kw.get("ns", 3), kw.get("nd", 3)
    x = np.zeros((3, 3), dtype=np.float32)
    nrm = np.zeros((3, 4), dtype=np.float32)
    res = capi.IcpResult()
    sn = None if kw.get("src_normals") in ("null", "null_entry") else nrm.ctypes.data_as(fp)
    dn = None if kw.get("dst_normals") in ("null", "null_entry") else nrm.ctypes.data_as(fp)
    assert capi.lib().tzr_icp_generalized(None, C.byref(p), kw.get("epsilon", 1e-3), x.ctypes.data_as(fp), ns, sn,
                                          x.ctypes.data_as(fp), nd, dn, None, C.byref(res), None) == \
        capi.TZR_ERR_INVALID_ARG


def test_chained_entry_refuses_null_icp_params():
    L = capi.lib()
    assert L.tzr_register_cloud_pairs_icp_generalized(None, None, None, 0, None, None, 0, None, None, None, None, None,
                                                      None, None, None, None, None, 1e-3, None) == \
        capi.TZR_ERR_INVALID_ARG


def test_chained_entry_takes_the_point_to_point_arguments_and_epsilon(header):
    m = re.search(r"int\s+tzr_register_cloud_pairs_icp\s*\(([^)]*)\)", header)
    q = re.search(r"int\s+tzr_register_cloud_pairs_icp_generalized\s*\(([^)]*)\)", header)
    a = [x.strip() for x in " ".join(m.group(1).split()).split(",")]
    b = [x.strip() for x in " ".join(q.group(1).split()).split(",")]
    assert b == a[:-1] + ["double epsilon"] + a[-1:]


def test_python_refuses_unknown_method_and_mismatched_normals():
    ctx = object.__new__(capi.Context)  # no device: both checks run before the library is called
    with pytest.raises(capi.TzrError):
        capi.Context.register_cloud_pairs_icp(ctx, [np.zeros((3, 3))], [(0, 0)], None, 0.1, method="plane_to_plane")
    with pytest.raises(capi.TzrError):
        capi.Context.icp_generalized_batch(ctx, [np.zeros((3, 3))], [np.zeros((3, 3))], [], [np.zeros((3, 4))], 0.1)
    with pytest.raises(capi.TzrError):
        capi.Context.icp_generalized_batch(ctx, [np.zeros((3, 3))], [np.zeros((3, 3))], [np.zeros((2, 4))],
                                           [np.zeros((3, 4))], 0.1)
