"""CPU checks of the ICP C-ABI (tzr_icp, tzr_icp_batch): the entry points are exported, declared in the header with the
argument lists the Python binding passes and listed among the symbols capi.lib() checks; the structs have the header's
layout; the defaults are ICPConvergenceCriteria's; malformed calls are refused before any device work."""
import ctypes as C
import importlib
import os
import re

import numpy as np
import pytest

capi = importlib.import_module("teaser-plusplus_b200.capi")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

ARGS = {
    "tzr_icp": ["ctx", "params", "src", "ns", "dst", "nd", "init", "result", "corr"],
    "tzr_icp_batch": ["ctx", "params", "B", "ns", "src", "nd", "dst", "init", "results", "corr"],
    "tzr_register_cloud_pairs_icp": ["ctx", "fparams", "params", "n_clouds", "n", "pts", "P", "pair_clouds",
                                     "tuple_seeds", "solutions", "status", "problem_index", "n_corr", "corr",
                                     "cliques", "global_scale", "icp", "icp_results"],
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
    assert name in capi._SYMBOLS and "tzr_icp_params_default" in capi._SYMBOLS
    assert len(getattr(capi.lib(), name).argtypes) == len(ARGS[name])
    assert re.search(r"void\s+tzr_icp_params_default\s*\(\s*tzr_icp_params\s*\*\s*p\s*\)", header)
    assert "#define TZR_ABI_VERSION 2" in header


def _fields(header, name):
    m = re.search(r"typedef struct %s \{(.*?)\} %s;" % (name, name), header, flags=re.S)
    assert m, name
    out = []
    for t, n, dim in re.findall(r"(double|int32_t|tzr_similarity)\s+(\w+)(?:\[(\d+)\])?;", m.group(1)):
        out.append((n, t, int(dim) if dim else None))
    return out


def test_struct_layouts(header):
    ct = {"double": C.c_double, "int32_t": C.c_int32, "tzr_similarity": capi.Similarity}
    for cname, cls in (("tzr_icp_params", capi.IcpParams), ("tzr_similarity", capi.Similarity),
                       ("tzr_icp_result", capi.IcpResult)):
        want = [(n, ct[t] * d if d else ct[t]) for n, t, d in _fields(header, cname)]
        got = cls._fields_
        assert [n for n, _ in want] == [n for n, _ in got], cname
        for (_, a), (_, b) in zip(want, got):
            assert C.sizeof(a) == C.sizeof(b) and getattr(a, "_type_", a) == getattr(b, "_type_", b), cname
    assert (C.sizeof(capi.IcpParams), C.sizeof(capi.Similarity), C.sizeof(capi.IcpResult)) == (32, 104, 136)
    assert capi.ICP_RESULT_DTYPE.itemsize == C.sizeof(capi.IcpResult)
    for name, _ in capi.IcpResult._fields_:
        assert capi.ICP_RESULT_DTYPE.fields[name][1] == getattr(capi.IcpResult, name).offset, name


def test_defaults():
    p = capi.IcpParams()
    p.max_correspondence_distance = 7.0
    p.reserved = 5
    capi.lib().tzr_icp_params_default(C.byref(p))
    # ICPConvergenceCriteria(relative_fitness=1e-6, relative_rmse=1e-6, max_iteration=30); no default distance
    assert (p.max_correspondence_distance, p.relative_fitness, p.relative_rmse, p.max_iteration, p.reserved) == \
        (0.0, 1e-6, 1e-6, 30, 0)


def _call_batch(ctx, p, B=1, ns=4, nd=4, init_scale=1.0):
    L = capi.lib()
    x = np.zeros((max(ns, 1), 3), dtype=np.float32)
    y = np.zeros((max(nd, 1), 3), dtype=np.float32)
    fp = C.POINTER(C.c_float)
    n_s = np.full(max(B, 1), ns, dtype=np.int32)
    n_d = np.full(max(B, 1), nd, dtype=np.int32)
    init = (capi.Similarity * max(B, 1))(*[capi.similarity(None) for _ in range(max(B, 1))])
    for s in init:
        s.scale = init_scale
    res = (capi.IcpResult * max(B, 1))()
    xs = (fp * max(B, 1))(*[x.ctypes.data_as(fp)] * max(B, 1))
    ys = (fp * max(B, 1))(*[y.ctypes.data_as(fp)] * max(B, 1))
    return L.tzr_icp_batch(ctx, C.byref(p), B, n_s.ctypes.data_as(C.POINTER(C.c_int32)), xs,
                           n_d.ctypes.data_as(C.POINTER(C.c_int32)), ys, init, res, None)


@pytest.mark.parametrize("case", ["null_ctx", "r_zero", "r_negative", "r_nan", "r_inf", "iter_negative", "B_zero",
                                  "ns_zero", "nd_zero", "scale_zero"])
def test_argument_checks_need_no_device(case):
    """Malformed calls return TZR_ERR_INVALID_ARG without a device (the context is NULL here, and every argument check
    runs before the device is touched)."""
    p = capi.icp_params(0.1)
    kw = {}
    if case == "r_zero":
        p.max_correspondence_distance = 0.0
    elif case == "r_negative":
        p.max_correspondence_distance = -1.0
    elif case == "r_nan":
        p.max_correspondence_distance = float("nan")
    elif case == "r_inf":
        p.max_correspondence_distance = float("inf")
    elif case == "iter_negative":
        p.max_iteration = -1
    elif case == "B_zero":
        kw["B"] = 0
    elif case == "ns_zero":
        kw["ns"] = 0
    elif case == "nd_zero":
        kw["nd"] = 0
    elif case == "scale_zero":
        kw["init_scale"] = 0.0
    assert _call_batch(None, p, **kw) == capi.TZR_ERR_INVALID_ARG
    if case in ("null_ctx", "r_zero", "r_nan", "iter_negative"):
        x = np.zeros((3, 3), dtype=np.float32)
        fp = C.POINTER(C.c_float)
        res = capi.IcpResult()
        assert capi.lib().tzr_icp(None, C.byref(p), x.ctypes.data_as(fp), 3, x.ctypes.data_as(fp), 3, None,
                                  C.byref(res), None) == capi.TZR_ERR_INVALID_ARG
